"""Piecewise streaming odometry at the shipped knobs: every sensor frame cut into 3 pieces and every piece registered as a scan of its own
(common/odom_mode 1, piecewise_number 3, mapping/maximum_histroy_buffer 400, mapping/init_accumulate_frames 50), through
Laser_mapping.process_new_frame (ll_mapper_process_frame), on a C3-style synthetic sequence of 100k-point frames with the leaves of
bench.py --workload c3.  Raw frames come from pinned host memory; host wall clock around each call.  Before timing, every piece of the first
frames is checked against the oracle (tests/piecewise_oracle.py).  The whole-frame path (process_new_scan) runs on the same frames in the same
process, alternating frame by frame, on a context and mapper of its own.  Prints the card, its power limit and SM clock beside the numbers.

    python scripts/piecewise_stream.py --frames 200 --warmup 5
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

N_PTS, PIECES, INIT, WINDOW, LINE, PLANE = 100000, 3, 50, 400, 0.05, 0.1


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.splitlines()[0].split(",")]))


def mapper(ctx, pieces):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping
    pipe = capi.PipelineCfg(pieces=pieces, use_piece=0, extractor_leaf_corner=LINE, extractor_leaf_surf=PLANE / 2, mapping_leaf_corner=LINE, mapping_leaf_surf=PLANE, whole_frame=1)
    return Laser_mapping(ctx, reg=capi.default_reg_state(mapping_init_accumulate_frames=INIT), pipeline=pipe, line_resolution=LINE, plane_resolution=PLANE,
                         maximum_history_size=WINDOW, reserve_map_points=1 << 22, reserve_store_points=1 << 23)


def front_end_launches(pieces):
    """Kernel launches of one frame's front end: a frame of <= 5 petals runs all of it and publishes nothing."""
    from loam_livox_b200 import synthetic as S
    from loam_livox_b200.registration import Context
    ctx = Context(0, max_scan_points=N_PTS, max_features=N_PTS)
    gm = mapper(ctx, pieces)
    raw = S.make_scan(N_PTS)[: N_PTS // 16].copy()   # 4 petals
    l0 = ctx.launches()
    assert gm.process_new_frame([raw], [100.0]) == []
    n = ctx.launches() - l0
    gm.close(); ctx.close()
    return n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--check", type=int, default=3, help="frames checked piece by piece against the oracle before timing")
    args = ap.parse_args()
    import torch
    from loam_livox_b200 import synthetic as S
    from loam_livox_b200.registration import Context
    from oracle import oracle as O
    import piecewise_oracle as PO
    n_total = args.frames + args.warmup
    poses = S.trajectory(n_scans=n_total, n_static=INIT // PIECES + 1, speed=1.0, zero_mean_yaw=True, y0=-1.6)
    ctx_p, ctx_s = Context(0, max_scan_points=N_PTS, max_features=N_PTS), Context(0, max_scan_points=N_PTS, max_features=N_PTS)
    gp, gs = mapper(ctx_p, PIECES), mapper(ctx_s, PIECES)
    om = O.Mapper(O.default_params(mapping_init_accumulate_frames=INIT, num_threads=8), threads=8, line_resolution=LINE, plane_resolution=PLANE,
                  extractor_leaf_corner=LINE, extractor_leaf_surf=PLANE / 2, maximum_history_size=WINDOW)
    pin = [torch.empty((N_PTS, 4), dtype=torch.float32).pin_memory() for _ in range(2)]
    t_frame, t_scan, regs, phases, checked = [], [], 0, [], 0
    for k in range(n_total):
        raw = S.make_scan(N_PTS, poses[k], seed=S.SEED + k)
        pin[k & 1].copy_(torch.from_numpy(raw))
        stamp = 100.0 + 0.1 * k
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = gp.process_new_frame([pin[k & 1].numpy()], [stamp])
        dt = time.perf_counter() - t0
        t0 = time.perf_counter()
        gs.process_new_scan(pin[k & 1].numpy(), stamp)
        ds = time.perf_counter() - t0
        if k < args.check:   # every piece against the oracle
            want = PO.process_frame(om, [raw], [stamp], PIECES)
            assert len(out) == len(want) == PIECES, k
            for i, ((res, st), (ost, oq, ot, L)) in enumerate(zip(out, want)):
                assert res.status == ost and (st.n_corner, st.n_surf) == (L["n_corner"], L["n_surf"]), (k, i)
                assert (st.map_corner, st.map_surf) == (L["map_corner"], L["map_surf"]), (k, i)
                assert np.linalg.norm(np.array(res.t_w_curr) - ot) < 1e-4 and S.quat_angle(np.array(res.q_w_curr), oq) < 1e-4, (k, i)
            checked += len(out)
        if k >= args.warmup:
            t_frame.append(dt); t_scan.append(ds)
            regs += sum(1 for res, _ in out if res.registered)
            phases += [(st.ms_front_end, st.ms_refresh, st.ms_register, st.ms_append) for _, st in out]
    ph = np.array(phases)
    line = {
        "gpu": gpu_info(),
        "frames": args.frames, "pieces": PIECES, "points_per_frame": N_PTS, "odom_mode": 1, "window": WINDOW, "init_accumulate_frames": INIT,
        "oracle_checked_pieces": checked,
        "piecewise_frames_per_s": len(t_frame) / float(np.sum(t_frame)),
        "piecewise_registrations_per_s": regs / float(np.sum(t_frame)),
        "whole_frame_scans_per_s": len(t_scan) / float(np.sum(t_scan)),
        "front_end_ms_per_frame_median": float(np.median(ph[::PIECES, 0])),
        "per_piece_ms_median": dict(zip(("front_end (charged to piece 0)", "refresh", "register", "append"), np.median(ph, axis=0).round(3).tolist())),
        "per_piece_ms_p99": dict(zip(("front_end (charged to piece 0)", "refresh", "register", "append"), np.percentile(ph, 99, axis=0).round(3).tolist())),
        "front_end_gpu_launches": {p: front_end_launches(p) for p in (1, 3, 16)},
        "frame_index": [int(gp.pose()[2]), int(gs.pose()[2])],
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
