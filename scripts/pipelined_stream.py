"""The sequence calls of the streaming mapper against the one-by-one calls, on recorded-data-style input (every frame already in pinned host
memory, as in a rosbag replay).

  frames: C3-style 100k-point frames at the shipped knobs (3 pieces, odom_mode 1, window 400, init_accumulate_frames 50), leaves of bench.py
          --workload c3: process_new_frame in a loop, process_new_frames in calls of 8, and process_new_frames in one call;
  scans:  the C3 scan stream (the same 100k-point scans, whole frame): process_new_scan in a loop against process_new_scans in one call.

Every arm first runs the whole sequence once on a fresh mapper and its outputs are compared with the one-by-one arm's (every ll_reg_result
field but the gpu_ms_* timings, every integer field of the stats, the final pose).  Then --rounds timed rounds, each arm on a fresh mapper of
its own context, the arm order alternating from round to round; host wall clock around each call.  Reports frames/s and scans/s, the per-phase
medians, the medians of gpu_ms_knn_all / gpu_ms_solve_all per registration (whether the front end under them slows the mapper's kernels) and
ms_front_end (one-by-one: enqueue + run of the front end; in a sequence: what is left of it on the host, i.e. its enqueue once it is hidden).
Prints the card, its power limit and SM clock beside the numbers.

    python scripts/pipelined_stream.py --frames 150 --rounds 2
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_PTS, PIECES, INIT, WINDOW, LINE, PLANE = 100000, 3, 50, 400, 0.05, 0.1


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.splitlines()[0].split(",")]))


def mapper(ctx):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping
    pipe = capi.PipelineCfg(pieces=PIECES, use_piece=0, extractor_leaf_corner=LINE, extractor_leaf_surf=PLANE / 2, mapping_leaf_corner=LINE, mapping_leaf_surf=PLANE, whole_frame=1)
    return Laser_mapping(ctx, reg=capi.default_reg_state(mapping_init_accumulate_frames=INIT), pipeline=pipe, line_resolution=LINE, plane_resolution=PLANE,
                         maximum_history_size=WINDOW, reserve_map_points=1 << 22, reserve_store_points=1 << 23)


def key(res, st):
    from loam_livox_b200 import capi
    val = lambda x: np.array(list(x) if isinstance(x, C.Array) else [x]).tobytes()  # noqa: E731
    return tuple(val(getattr(res, f)) for f, _ in capi.RegResult._fields_ if not f.startswith("gpu_ms")) + \
        tuple(getattr(st, f) for f, t in capi.MapperStats._fields_ if t is C.c_int)


def run_arm(ctx, arm, frames, stamps):
    """One whole sequence on a fresh mapper: (seconds in the calls, [(res, stats) per registered entry, in order], final pose)."""
    gm = mapper(ctx)
    out, secs = [], 0.0
    import torch
    torch.cuda.synchronize()
    if arm == "frame":
        for f, t in zip(frames, stamps):
            t0 = time.perf_counter(); r = gm.process_new_frame([f], [t]); secs += time.perf_counter() - t0
            out += r
    elif arm.startswith("frames"):
        chunk = int(arm[6:]) if arm != "frames" else len(frames)
        for i in range(0, len(frames), chunk):
            t0 = time.perf_counter(); r = gm.process_new_frames([[f] for f in frames[i:i + chunk]], [[t] for t in stamps[i:i + chunk]]); secs += time.perf_counter() - t0
            out += [e for fr in r for e in fr]
    elif arm == "scan":
        for f, t in zip(frames, stamps):
            t0 = time.perf_counter(); r = gm.process_new_scan(f, t); secs += time.perf_counter() - t0
            out.append(r)
    elif arm == "scans":
        t0 = time.perf_counter(); out = gm.process_new_scans(list(frames), list(stamps)); secs += time.perf_counter() - t0
    pose = gm.pose()
    gm.close()
    return secs, out, (pose[0].tobytes(), pose[1].tobytes(), pose[2])


def summary(n_inputs, secs, out):
    ph = np.array([(s.ms_front_end, s.ms_refresh, s.ms_register, s.ms_append) for _, s in out])
    reg = [r for r, _ in out if r.registered]
    fe = ph[::PIECES, 0] if len(out) == PIECES * n_inputs else ph[:, 0]
    return {"inputs_per_s": n_inputs / secs,
            "ms_front_end_median": float(np.median(fe)),
            "per_entry_ms_median": dict(zip(("front_end", "refresh", "register", "append"), np.median(ph, axis=0).round(3).tolist())),
            "gpu_ms_knn_all_median": float(np.median([r.gpu_ms_knn_all for r in reg])) if reg else None,
            "gpu_ms_solve_all_median": float(np.median([r.gpu_ms_solve_all for r in reg])) if reg else None,
            "registrations": len(reg)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=150)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    import torch
    from loam_livox_b200 import synthetic as S
    from loam_livox_b200.registration import Context
    poses = S.trajectory(n_scans=args.frames, n_static=INIT // PIECES + 1, speed=1.0, zero_mean_yaw=True, y0=-1.6)
    frames = [torch.from_numpy(S.make_scan(N_PTS, p, seed=S.SEED + k)).pin_memory().numpy() for k, p in enumerate(poses)]
    stamps = [100.0 + 0.1 * k for k in range(args.frames)]
    groups = {"frames": ["frame", "frames8", "frames"], "scans": ["scan", "scans"]}
    ctxs = {a: Context(0, max_scan_points=N_PTS, max_features=N_PTS) for g in groups.values() for a in g}
    # outputs first: every arm against its group's one-by-one arm
    for g, arms in groups.items():
        _, ref, ref_pose = run_arm(ctxs[arms[0]], arms[0], frames, stamps)
        for a in arms[1:]:
            _, out, pose = run_arm(ctxs[a], a, frames, stamps)
            assert [key(*e) for e in out] == [key(*e) for e in ref] and pose == ref_pose, f"{a} differs from {arms[0]}"
    results = {a: [] for a in ctxs}
    for rnd in range(args.rounds):
        for g, arms in groups.items():
            for a in (arms if rnd % 2 == 0 else arms[::-1]):
                secs, out, _ = run_arm(ctxs[a], a, frames, stamps)
                results[a].append(summary(args.frames, secs, out))
    line = {"gpu": gpu_info(), "frames": args.frames, "points": N_PTS, "pieces": PIECES, "window": WINDOW, "init_accumulate_frames": INIT, "rounds": args.rounds,
            "outputs_identical": True, "arms": results}
    print(json.dumps(line))
    for c in ctxs.values():
        c.close()


if __name__ == "__main__":
    main()
