"""What loop feedback costs the streaming mapper (DESIGN.md §4.6.2): the synthetic-room stream that returns to its start twice
(scripts/loop_closure_profile.py's), loop closure on with max_loops 2 and gap 4, run with feedback off and on, alternating over --rounds rounds
after one warm-up round, on fresh mappers of one context.  Every step is one ll_mapper_process_scan call, timed by the host clock around the call
(it returns the step's results, so it ends in a device synchronisation).

Reported: the first loop's closing step (the same step both ways), the median over the rounds of its time with feedback on minus off; the
closing steps of each run's later loops (feedback changes the odometry after the first loop, so later loops may close at other steps) with
their median times; the median added per step over the steps after the first loop that close no loop either way; the correction kernel alone, lc_window_correct_kernel's device time from
torch.profiler (CUDA activities) in a separate run, with the points it moved; the worst distance from the synthetic truth after the first loop
both ways.  Prints the card and its power limit, read in the same run, and one JSON line.

    python scripts/loop_feedback_profile.py --rounds 3 --points 24000
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from loop_closure_profile import CFG, mapper, stream  # noqa: E402
from mapper_checkpoint import gpu_info  # noqa: E402


def run(ctx, poses, raws, stamps, feedback):
    """per-step ms, the closing frame indices, the worst error after the first loop, points in the windows at each correction"""
    from loam_livox_b200 import capi
    m = mapper(ctx, poses[0])
    try:
        m.set_loop_closure(**CFG)
        m.set_loop_policy(2, 4)
        m.set_loop_feedback(feedback)
        ms, ts = [], []
        for r, s in zip(raws, stamps):
            t0 = time.perf_counter()
            res, _ = m.process_new_scan(r, s)
            ms.append((time.perf_counter() - t0) * 1e3)
            ts.append(np.array(res.t_w_curr))
        log, _ = m.loop_log()
        end = {e.keyframe: e.ending_frame_idx for e in log if e.kind == capi.LL_LOOP_KEYFRAME}
        closing = [end[e.keyframe] for e in log if e.kind == capi.LL_LOOP_CLOSED]
        worst = max(float(np.linalg.norm(ts[k] - poses[k].t)) for k in range(len(ts)) if closing and k + 1 > closing[0])
        return ms, closing, worst
    finally:
        m.close()


def kernel_time(ctx, poses, raws, stamps):
    """the correction kernel's launches (device ms each) from torch.profiler over one feedback run"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(ctx, poses, raws, stamps, True)
        torch.cuda.synchronize()
    return [e.device_time_total / 1e3 for e in prof.events() if e.name.startswith("_Z24lc_window_correct_kernel") or e.name.startswith("lc_window_correct_kernel")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--points", type=int, default=24000)
    a = ap.parse_args()
    import torch
    torch.cuda.init()
    from loam_livox_b200.registration import Context
    info = gpu_info()
    ctx = Context(0, max_scan_points=60000, max_features=400000)
    poses, raws, stamps = stream(a.points, 6100)
    run(ctx, poses, raws, stamps, False)   # warm-up
    per = {False: [], True: []}
    for _ in range(a.rounds):
        for fb in (False, True):
            per[fb].append(run(ctx, poses, raws, stamps, fb))
    c_on, c_off = per[True][0][1], per[False][0][1]
    assert all(r[1] == c_on for r in per[True]) and all(r[1] == c_off for r in per[False]) and c_on[0] == c_off[0], "the loops closed at other steps"
    off = np.array([r[0] for r in per[False]]); on = np.array([r[0] for r in per[True]])
    f0 = c_on[0]
    added = float(np.median(on[:, f0 - 1] - off[:, f0 - 1]))
    later = [k for k in range(off.shape[1]) if k + 1 > f0 and k + 1 not in c_on and k + 1 not in c_off]
    kt = kernel_time(ctx, poses, raws, stamps)
    ctx.close()
    out = dict(gpu=info, points=a.points, rounds=a.rounds, closing_frames=dict(on=c_on, off=c_off), first_closing_step_added_ms=added,
               first_closing_step_off_ms=float(np.median(off[:, f0 - 1])),
               closing_step_ms=dict(on={f: float(np.median(on[:, f - 1])) for f in c_on}, off={f: float(np.median(off[:, f - 1])) for f in c_off}),
               later_step_added_ms_median=float(np.median(on[:, later] - off[:, later])), kernel_ms=kt,
               worst_error_after_first_loop_m=dict(off=per[False][0][2], on=per[True][0][2]))
    print(f"{info['name']} at a power limit of {info['power.limit']}: closing steps on {c_on} off {c_off}, first closing step +{added:.3f} ms "
          f"with feedback; kernel {kt} ms; "
          f"worst error after the first loop off {out['worst_error_after_first_loop_m']['off']:.4f} m, on {out['worst_error_after_first_loop_m']['on']:.4f} m")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
