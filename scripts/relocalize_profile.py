#!/usr/bin/env python
"""Relocalization timing (ll_reloc_index_build, ll_reloc_scores, ll_relocalize): index build, scoring, peak selection and refinement, each timed
with a host clock around work that ends in a device synchronise (every entry point synchronises before it returns), on

  c2      the C2 map (0.5 M corner + 4.5 M surface points) and a 100k-point scan at a known pose, the window covering the whole room
          (x -1 ... 39, y -5 ... 5 at 1 m, z at the truth, 36 yaws at 10 degrees: 16 236 hypotheses);
  stream  the whole map of a mapper saved after a C3-style stream (ll_mapper_whole_map), a later scan of the same stream, the same window.

Peak selection is the part of ll_relocalize that is neither scoring nor refinement: its time is the relocalization's minus the scoring call's
minus the refinement (the batch's gpu_ms_total).  Prints one JSON line per case with hypotheses x points per second and the card's name and
power limit.  Needs a GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from loam_livox_b200 import synthetic as S  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=20).stdout.strip()
        name, power = [x.strip() for x in out.splitlines()[0].split(",")]
        return name, power
    except Exception:
        return "unknown", "unknown"


def features(ctx, raw, stamp, leaves):
    from loam_livox_b200.registration import Livox_laser, voxel_grid_filter
    lx = Livox_laser(ctx)
    lx.extract_laser_features(raw, stamp)
    c, s, _ = lx.get_features(0.0, 1.0)
    return (voxel_grid_filter(ctx, voxel_grid_filter(ctx, c, leaves[0]), leaves[1]), voxel_grid_filter(ctx, voxel_grid_filter(ctx, s, leaves[2]), leaves[3]))


def timed(f, reps):
    f()   # warm-up: module loads
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = f()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), r


def run_case(name, ctx, m, fc, fs, truth, args):
    from loam_livox_b200.registration import RelocIndex, reloc_scores, relocalize, voxel_grid_filter, window_lattice, yaw_circle
    window = ((-1.0, 39.0, args.step), (-5.0, 5.0, args.step), (truth.t[2], truth.t[2], 0.0))
    ms_index, idx = timed(lambda: RelocIndex(ctx, m, args.res, args.dilate, 1 << 18), args.reps)
    pts = voxel_grid_filter(ctx, np.concatenate([fc, fs]), args.score_leaf)
    rot = yaw_circle(10.0)
    t0, step, nt = window_lattice(window)
    H = rot.shape[0] * int(np.prod(nt))
    ms_score, _ = timed(lambda: reloc_scores(ctx, idx, pts, rot, t0, step, nt), args.reps)
    ms_reloc, out = timed(lambda: relocalize(ctx, m, idx, fc, fs, window=window, yaw_step_deg=10.0, k=args.k, score_pts=pts), args.reps)
    ms_refine = float(out["refined"][0].gpu_ms_total) if out["refined"] else 0.0
    b = out["best"]
    err_t = err_a = None
    if b >= 0:
        r = out["refined"][b]
        err_t = float(np.linalg.norm(np.array(r.t_w_curr) - truth.t))
        err_a = float(np.degrees(S.quat_angle(np.array(r.q_w_curr), truth.q)))
    dims = idx.read()[0].tolist()
    return {"case": name, "map_points": [m.size(0), m.size(1)], "features": [int(fc.shape[0]), int(fs.shape[0])], "score_points": int(pts.shape[0]),
            "hypotheses": H, "grid": dims, "res": args.res, "dilate": args.dilate, "k": args.k, "candidates": len(out["candidates"]), "best": b,
            "best_err_m": err_t, "best_err_deg": err_a,
            "ms_index_build": ms_index, "ms_scores_call": ms_score, "ms_relocalize": ms_reloc, "ms_refine_gpu": ms_refine,
            "ms_peaks_and_overhead": ms_reloc - ms_score - ms_refine,
            "hyp_points_per_s_scoring_call": H * pts.shape[0] / (ms_score * 1e-3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--res", type=float, default=0.2)
    ap.add_argument("--dilate", type=int, default=1)
    ap.add_argument("--score-leaf", type=float, default=0.5)
    ap.add_argument("--k", type=int, default=8)
    ap.add_argument("--step", type=float, default=1.0, help="lattice step in x and y (m)")
    ap.add_argument("--stream-scans", type=int, default=60)
    args = ap.parse_args()
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Context, Laser_mapping, Map
    name, power = card()
    ctx = Context(0, max_scan_points=200000, max_features=400000)
    # c2
    mc, ms = S.make_map(500_000, 4_500_000)
    m = Map(ctx, mc, ms)
    truth = S.Pose(S.quat_from_euler(0.0, 0.0, np.radians(0.5)), np.array([10.05, -0.97, 0.1]))   # the pose tests/test_gpu_relocalize.py finds in a one-pitch window
    fc, fs = features(ctx, S.make_scan(100_000, truth, seed=S.SEED + 77), 100.0, (0.1, 0.2, 0.2, 0.4))
    print(json.dumps(dict(run_case("c2", ctx, m, fc, fs, truth, args), gpu=name, power_limit=power)), flush=True)
    m.release()
    # a mapper image of a C3-style stream, its whole map
    n = args.stream_scans
    poses = S.trajectory(n_scans=n + 20, n_static=4, speed=1.0)
    pipe = capi.PipelineCfg(pieces=3, use_piece=0, extractor_leaf_corner=0.05, extractor_leaf_surf=0.05, mapping_leaf_corner=0.05, mapping_leaf_surf=0.1, whole_frame=1)
    p0 = poses[0]   # the mapper's world frame is the synthetic one
    gm = Laser_mapping(ctx, reg=capi.default_reg_state(mapping_init_accumulate_frames=3, q_w_last=p0.q, t_w_last=p0.t, q_w_curr=p0.q, t_w_curr=p0.t), pipeline=pipe, line_resolution=0.05, plane_resolution=0.1, matching_mode=0,
                       maximum_history_size=400)
    for k in range(n):
        gm.process_new_scan(S.make_scan(100_000, poses[k], seed=S.SEED + k), 100.0 + 0.1 * k)
    img = gm.save()
    gm.close()
    ctx2 = Context(0, max_scan_points=200000, max_features=400000)
    lm = Laser_mapping.load(ctx2, img)
    wm = lm.whole_map()
    k = n + 19
    fc, fs = features(ctx2, S.make_scan(100_000, poses[k], seed=S.SEED + k), 100.0 + 0.1 * k, (0.1, 0.2, 0.2, 0.4))
    print(json.dumps(dict(run_case("stream", ctx2, wm, fc, fs, poses[k], args), image_bytes=len(img), gpu=name, power_limit=power)), flush=True)
    wm.release(); lm.close(); ctx2.close(); ctx.close()


if __name__ == "__main__":
    main()
