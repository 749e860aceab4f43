#!/usr/bin/env python
"""Relocalization by class-aware distance fields (ll_reloc_field_build, ll_relocalize_field) against the occupancy relocalization
(ll_relocalize) on the same hypotheses, each phase timed with a host clock around work that ends in a device synchronise (every entry point
synchronises before it returns; medians after one warm-up), on

  c2          the C2 map (0.5 M corner + 4.5 M surface points) and a 100k-point scan at (10.05, -0.97, 0.1), yaw 0.5 deg;
  c2_off      the same map and a scan at (10.55, -0.47, 0.1), yaw 5.5 deg: about 0.65 m and 4.5 deg from the nearest hypothesis;
  stream      the whole map of a mapper saved after a C3-style stream (ll_mapper_whole_map) and a later scan of the same stream;

every case over the whole room: x -1 ... 39, y -5 ... 5 at 1 m, z at the truth, 36 yaws at 10 deg (16 236 hypotheses), K = 8, the fine
search of registration.fine_search (yaw +-5 deg at 1 deg, x / y +-fine_t_half coarse steps at 0.1 m: 10 571 hypotheses per candidate at the
default 1.5).

Phases: the field build; the coarse scoring call (ll_reloc_field_scores over the coarse lattice, with its uploads and the copy back); the fine
search (one ll_reloc_field_scores call per candidate's group, so it includes K uploads and synchronises); the refinement (the batch's
gpu_ms_total); the rest of ll_relocalize_field (peaks, picks, verify and host work) = total - coarse - fine - refinement.  Prints one JSON line per
case and field setting, with the card's name and power limit.  Needs a GPU.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from loam_livox_b200 import synthetic as S  # noqa: E402
import reloc_field_reference as F  # noqa: E402  (the fine groups' host formulas)


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
    r = f()   # warm-up: module loads
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = f()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), r


def err(out, truth):
    b = out["best"]
    if b < 0:
        return None, None
    r = out["refined"][b]
    return float(np.linalg.norm(np.array(r.t_w_curr) - truth.t)), float(np.degrees(S.quat_angle(np.array(r.q_w_curr), truth.q)))


def run_case(name, ctx, m, fc, fs, truth, res, trunc, half, args):
    from loam_livox_b200.registration import (RelocField, RelocIndex, fine_search, reloc_field_scores, relocalize, relocalize_field, voxel_grid_filter,
                                              window_lattice, yaw_circle)
    window = ((-1.0, 39.0, 1.0), (-5.0, 5.0, 1.0), (truth.t[2], truth.t[2], 0.0))
    rot = yaw_circle(10.0)
    t0, step, nt = window_lattice(window)
    H = rot.shape[0] * int(np.prod(nt))
    sp = (voxel_grid_filter(ctx, fc, args.score_leaf), voxel_grid_filter(ctx, fs, args.score_leaf))
    n_pts = int(sp[0].shape[0] + sp[1].shape[0])
    ms_build, fld = timed(lambda: RelocField(ctx, m, res, trunc, 1 << 18), args.reps)
    ms_coarse, _ = timed(lambda: reloc_field_scores(ctx, fld, sp[0], sp[1], rot, t0, step, nt), args.reps)
    ms_total, out = timed(lambda: relocalize_field(ctx, m, fld, fc, fs, window=window, yaw_step_deg=10.0, k=args.k, score_pts=sp, fine_t_half=half), args.reps)
    dq, fstep, fnt = fine_search(10.0, window, fine_t_half=half)
    groups = [F.fine_group(c["q"], c["t"], dq, fstep, fnt) for c in out["candidates"]]
    ms_fine, _ = timed(lambda: [reloc_field_scores(ctx, fld, sp[0], sp[1], g[0], g[1], fstep, fnt) for g in groups], args.reps)
    ms_refine = float(out["refined"][0].gpu_ms_total) if out["refined"] else 0.0
    H_f = len(groups) * dq.shape[0] * int(np.prod(fnt))
    e_t, e_r = err(out, truth)
    # the occupancy relocalization on the same hypotheses (its defaults: 0.2 m, dilate 1, both classes' VoxelGrid at 0.5 m)
    idx = RelocIndex(ctx, m, 0.2, 1, 1 << 16)
    ms_occ, occ = timed(lambda: relocalize(ctx, m, idx, fc, fs, window=window, yaw_step_deg=10.0, k=args.k), args.reps)
    o_t, o_r = err(occ, truth)
    idx.close()
    cands = [{"t": [round(v, 3) for v in c["t"]], "score": c["score"], "fine_t": [round(v, 3) for v in c["fine_t"]], "fine_score": c["fine_score"],
              "verify": c["verify_score"], "status": out["refined"][j].status} for j, c in enumerate(out["candidates"])]
    row = {"case": name, "map_points": [m.size(0), m.size(1)], "features": [int(fc.shape[0]), int(fs.shape[0])], "score_points": [int(sp[0].shape[0]), int(sp[1].shape[0])],
           "res": res, "trunc": trunc, "fine_t_half": half, "grid": fld.read(0)[0].tolist(), "hypotheses": H, "fine_hypotheses": H_f, "k": args.k, "best": out["best"],
           "best_err_m": e_t, "best_err_deg": e_r, "occupancy_best_err_m": o_t, "occupancy_best_err_deg": o_r,
           "ms_field_build": ms_build, "ms_coarse_call": ms_coarse, "ms_fine_calls": ms_fine, "ms_refine_gpu": ms_refine,
           "ms_peaks_picks_verify_overhead": ms_total - ms_coarse - ms_fine - ms_refine, "ms_total": ms_total, "ms_occupancy_relocalize": ms_occ,
           "hyp_points_per_s_coarse_call": H * n_pts / (ms_coarse * 1e-3), "hyp_points_per_s_fine_calls": H_f * n_pts / (ms_fine * 1e-3), "candidates": cands}
    fld.close()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--fields", default="0.2:2", help="comma-separated res:trunc settings of the field")
    ap.add_argument("--fine-half", default="1.5", help="comma-separated fine translation half-widths, in coarse steps")
    ap.add_argument("--score-leaf", type=float, default=0.5)
    ap.add_argument("--k", type=int, default=8)
    ap.add_argument("--stream-scans", type=int, default=60)
    args = ap.parse_args()
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Context, Laser_mapping, Map
    name, power = card()
    fields = [(float(a), int(b), float(h)) for a, b in (x.split(":") for x in args.fields.split(",")) for h in args.fine_half.split(",")]
    ctx = Context(0, max_scan_points=200000, max_features=400000)
    mc, ms = S.make_map(500_000, 4_500_000)
    m = Map(ctx, mc, ms)
    for case, (x, y, yaw) in (("c2", (10.05, -0.97, 0.5)), ("c2_off", (10.55, -0.47, 5.5))):
        truth = S.Pose(S.quat_from_euler(0.0, 0.0, np.radians(yaw)), np.array([x, y, 0.1]))
        fc, fs = features(ctx, S.make_scan(100_000, truth, seed=S.SEED + 77), 100.0, (0.1, 0.2, 0.2, 0.4))
        for res, trunc, half in fields:
            print(json.dumps(dict(run_case(case, ctx, m, fc, fs, truth, res, trunc, half, args), gpu=name, power_limit=power)), flush=True)
    m.release()
    n = args.stream_scans
    poses = S.trajectory(n_scans=n + 20, n_static=4, speed=1.0)
    pipe = capi.PipelineCfg(pieces=3, use_piece=0, extractor_leaf_corner=0.05, extractor_leaf_surf=0.05, mapping_leaf_corner=0.05, mapping_leaf_surf=0.1, whole_frame=1)
    p0 = poses[0]   # the mapper's world frame is the synthetic one
    gm = Laser_mapping(ctx, reg=capi.default_reg_state(mapping_init_accumulate_frames=3, q_w_last=p0.q, t_w_last=p0.t, q_w_curr=p0.q, t_w_curr=p0.t), pipeline=pipe,
                       line_resolution=0.05, plane_resolution=0.1, matching_mode=0, maximum_history_size=400)
    for k in range(n):
        gm.process_new_scan(S.make_scan(100_000, poses[k], seed=S.SEED + k), 100.0 + 0.1 * k)
    img = gm.save()
    gm.close()
    ctx2 = Context(0, max_scan_points=200000, max_features=400000)
    lm = Laser_mapping.load(ctx2, img)
    wm = lm.whole_map()
    k = n + 19
    fc, fs = features(ctx2, S.make_scan(100_000, poses[k], seed=S.SEED + k), 100.0 + 0.1 * k, (0.1, 0.2, 0.2, 0.4))
    for res, trunc, half in fields:
        print(json.dumps(dict(run_case("stream", ctx2, wm, fc, fs, poses[k], res, trunc, half, args), image_bytes=len(img), gpu=name, power_limit=power)), flush=True)
    wm.release(); lm.close(); ctx2.close(); ctx.close()


if __name__ == "__main__":
    main()
