"""What loop closure costs the streaming mapper (DESIGN.md §4.6): one synthetic-room stream that returns to its start twice (out along the room,
back, out again and back; tests/test_gpu_loop_policy.py's stream), run three ways on fresh mappers of one context:

  off        loop closure off;
  reference  loop closure on with the default policy (the reference's first loop, then stop);
  multi      loop closure on with --max-loops / --gap (ll_mapper_set_loop_policy).

Keyframes of 6 scans opened every 2, the search of tests/test_gpu_loop_closure.py's parity test.  Every step is one ll_mapper_process_scan call,
timed by the host clock around the call (it returns the step's results, so it ends in a device synchronisation).  Reported per run: the time added
per step over the off run at the same step (median and p99 over the steps of every round), the latency of each step that closes a loop and the
part of it spent in the pose-graph solve (the solve's SM clock cycles, ll_pg_summary::cycles_total, at the card's maximum SM clock, so a lower
bound on its time when the clock runs lower), and the device memory the run adds (cudaMemGetInfo through torch, against the reading before
its mapper's loop closure) after ll_mapper_set_loop_closure and at the end.  The runs alternate over --rounds rounds after one warm-up round.  Prints the card and its power limit, read in the same run, and one JSON line.

    python scripts/loop_closure_profile.py --rounds 3 --points 24000
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
from mapper_checkpoint import gpu_info  # noqa: E402

CFG = dict(scans_of_each_keyframe=6, scans_between_two_keyframe=2, map_alignment_inlier_threshold=0.35, reserve_map_points=1 << 21,
           reserve_history_points=1 << 20, reserve_keyframes=64, loop=dict(minimum_keyframe_differen=36, avail_ratio_plane=0.02, avail_ratio_line=0.005))


def stream(n_points, seed):
    from loam_livox_b200 import synthetic as S
    xs = [0.3 + 0.15 * k for k in range(40)] + [0.3 + 0.15 * (39 - k) for k in range(40)]
    xs = xs + xs[1:]
    poses = [S.Pose(np.array([1.0, 0.0, 0.0, 0.0]), np.array([x, 0.2, 0.0])) for x in xs]
    return poses, [S.make_scan(n_points, p, seed=seed + k) for k, p in enumerate(poses)], [100.0 + 0.1 * k for k in range(len(poses))]


def mapper(ctx, p0):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping
    pipe = capi.PipelineCfg(pieces=3, use_piece=0, extractor_leaf_corner=0.1, extractor_leaf_surf=0.2, mapping_leaf_corner=0.1, mapping_leaf_surf=0.4, whole_frame=1)
    st = capi.default_reg_state(mapping_init_accumulate_frames=3, q_w_last=p0.q, t_w_last=p0.t, q_w_curr=p0.q, t_w_curr=p0.t)
    return Laser_mapping(ctx, reg=st, pipeline=pipe, matching_mode=0, maximum_history_size=400)


def used_mib():
    import torch
    free, total = torch.cuda.mem_get_info()
    return (total - free) / 2**20


def run(ctx, poses, raws, stamps, policy):
    """policy None: loop closure off; else (max_loops, gap).  Returns per-step ms, the closing steps, the memory readings."""
    from loam_livox_b200 import capi
    m = mapper(ctx, poses[0])
    mem = {"before": used_mib()}   # the device is shared: what this run adds is reported, not the total
    if policy is not None:
        m.set_loop_closure(**CFG)
        m.set_loop_policy(*policy)
        mem["set_loop_closure"] = used_mib() - mem["before"]
    ms = []
    for raw, st in zip(raws, stamps):
        t0 = time.perf_counter()
        m.process_new_scan(raw, st)
        ms.append(1e3 * (time.perf_counter() - t0))
    mem["end"] = used_mib() - mem["before"]
    closing = []
    if policy is not None:
        log, _ = m.loop_log()
        end = {e.keyframe: e.ending_frame_idx for e in log if e.kind == capi.LL_LOOP_KEYFRAME}
        closing = [dict(step=end[e.keyframe] - 1, keyframe=e.keyframe, his=e.his, cycles=e.summary.cycles_total, border=e.summary.border_nodes,
                        iterations=e.summary.iterations) for e in log if e.kind == capi.LL_LOOP_CLOSED]
    m.close()
    return np.array(ms), closing, mem


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--points", type=int, default=24000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--max-loops", type=int, default=2)
    ap.add_argument("--gap", type=int, default=4)
    ap.add_argument("--seed", type=int, default=6100)
    a = ap.parse_args()
    from loam_livox_b200 import synthetic as S
    from loam_livox_b200.registration import Context
    info = gpu_info()
    sm_mhz = float(info["clocks.max.sm"].split()[0])
    poses, raws, stamps = stream(a.points, S.SEED + a.seed)
    ctx = Context(0, max_scan_points=60000, max_features=400000)
    runs = {"off": None, "reference": (1, 0), "multi": (a.max_loops, a.gap)}
    for name, pol in runs.items():   # warm-up round: modules, allocations
        run(ctx, poses, raws, stamps, pol)
    steps = {k: [] for k in runs}
    closing, mem = {k: [] for k in runs}, {}
    for r in range(a.rounds):
        for name, pol in runs.items():
            ms, cl, mm = run(ctx, poses, raws, stamps, pol)
            steps[name].append(ms)
            closing[name].append(cl)
            mem[name] = mm
    out = {"card": info["name"], "power_limit": info["power.limit"], "sm_clock_max_mhz": sm_mhz, "steps": len(raws), "points": a.points,
           "rounds": a.rounds, "policy_multi": [a.max_loops, a.gap]}
    off = np.stack(steps["off"])
    for name in ("reference", "multi"):
        s = np.stack(steps[name])
        added = (s - off).ravel()
        cl = []
        for k, c in enumerate(closing[name][0]):
            lat = [float(steps[name][r][c["step"]]) for r in range(a.rounds)]
            add = [float(steps[name][r][c["step"]] - steps["off"][r][c["step"]]) for r in range(a.rounds)]
            solve = [closing[name][r][k]["cycles"] / (sm_mhz * 1e3) for r in range(a.rounds)]
            cl.append(dict(loop=k + 1, keyframe=c["keyframe"], his=c["his"], border=c["border"], iterations=c["iterations"], step_ms=float(np.median(lat)),
                           added_ms=float(np.median(add)), solve_ms=float(np.median(solve)), solve_share=float(np.median(solve) / np.median(lat))))
        out[name] = dict(added_ms_median=float(np.median(added)), added_ms_p99=float(np.percentile(added, 99)), step_ms_median=float(np.median(s)),
                         closing=cl, mem_mib=mem[name])
        print(f"{name}: added per step median {out[name]['added_ms_median']:.3f} ms, p99 {out[name]['added_ms_p99']:.3f} ms")
        for c in cl:
            print(f"  loop {c['loop']} (keyframe {c['keyframe']} -> {c['his']}, border {c['border']}): closing step {c['step_ms']:.2f} ms "
                  f"(+{c['added_ms']:.2f} ms), solve {c['solve_ms']:.2f} ms = {100 * c['solve_share']:.1f} %")
        print(f"  device memory added (MiB): after set_loop_closure {mem[name]['set_loop_closure']:.1f}, at the end {mem[name]['end']:.1f}")
    out["off"] = dict(step_ms_median=float(np.median(off)), mem_mib=mem["off"])
    print(f"off: step median {out['off']['step_ms_median']:.3f} ms; {info['name']} at a {info['power.limit']} power limit")
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
