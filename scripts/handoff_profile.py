#!/usr/bin/env python
"""The gap between the front end and the registration of a C2 step (bench.py's headline workload: one 100k-pt scan through ll_scan_to_pose
against the 5M-point map), under torch.profiler (CUDA activity only, a run of its own).

Per profiled step: the end of the last kernel before the query sort's key kernel (the front end's last kernel, or the kernel that moves its
features into the registration's arrays) and the start of the key kernel.  The gap between them is the time the GPU runs no kernel of this
step between the front end and the registration; with a host read of the counts in between, it holds the read-back, the host's wake-up and the
enqueue of the registration.  Also the per-launch times of knn_blocks_kernel and lm_solve_kernel and the step's span.  The card's name and
power limit are read in the same run.  Prints a table and one JSON line.

    python scripts/handoff_profile.py --steps 60 --label new
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import bench  # noqa: E402
from solver_profile import gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60, help="profiled steps (cycling through the distinct scans)")
    ap.add_argument("--warmup", type=int, default=3, help="steps of each distinct scan before the profiled ones")
    ap.add_argument("--label", default="", help="tag printed with the results (e.g. which build)")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Context, Map, scan_to_pose

    device = 0
    torch.cuda.set_device(device)
    mc, ms, scans, guesses, _ = bench.make_inputs(0, "c2")
    ctx = Context(device, max_scan_points=bench.N_SCAN, max_features=bench.N_SCAN)
    m = Map(ctx, mc, ms)
    pc = capi.PipelineCfg(**bench.PIPE)
    states = [capi.default_reg_state(q_w_last=g.q, t_w_last=g.t, q_w_curr=g.q, t_w_curr=g.t) for g in guesses]
    dev_scans = [torch.from_numpy(s).cuda() for s in scans]
    stream = torch.cuda.ExternalStream(ctx.stream(), device=device)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    nd = len(scans)

    def step(k):
        return scan_to_pose(ctx, m, dev_scans[k].data_ptr(), 100.0 + 0.1 * k, pc, states[k], where=capi.LL_DEVICE, n=bench.N_SCAN, fmt=capi.LL_FMT_XYZI16)

    for _ in range(args.warmup):
        for k in range(nd):
            step(k)
    torch.cuda.synchronize()
    info = gpu_info(device)
    gap, span, knn, solve = [], [], [], []
    for i in range(args.steps):
        with torch.cuda.stream(stream):
            flush.zero_()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            res, _, _ = step(i % nd)
            torch.cuda.synchronize()
        assert res.status == 1 and res.registered == 1, (i, res.status)
        ks = sorted([(e.time_range.start, e.time_range.end, e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                     and e.time_range.end > e.time_range.start and "Memcpy" not in e.name and "Memset" not in e.name])
        ks = [k for k in ks if "elementwise" not in k[2] and "fill" not in k[2].lower()]   # (the L2 flush)
        key = next(k for k in ks if "query_key_kernel" in k[2])
        before = [k for k in ks if k[0] < key[0]]
        gap.append(key[0] - max(e for _, e, _ in before))
        span.append(max(e for _, e, _ in ks) - ks[0][0])
        knn += [e - s for s, e, n in ks if "knn_blocks_kernel" in n]
        solve += [e - s for s, e, n in ks if "lm_solve_kernel" in n]
    out = {"label": args.label, "gpu": info["name"], "power_limit_w": info["power_limit_w"], "steps": args.steps,
           "gap_us_median": float(np.median(gap)), "gap_us_p10": float(np.percentile(gap, 10)), "gap_us_p90": float(np.percentile(gap, 90)),
           "step_span_us_median": float(np.median(span)),
           "knn_us_per_launch_median": float(np.median(knn)), "knn_launches_per_step": len(knn) / args.steps,
           "solve_us_per_launch_median": float(np.median(solve)), "solve_launches_per_step": len(solve) / args.steps}
    print(f"handoff profile {args.label}: {info['name']}, power limit {info['power_limit_w']:.0f} W, {args.steps} profiled steps")
    print(f"  front end -> query sort gap: median {out['gap_us_median']:.1f} us (p10 {out['gap_us_p10']:.1f}, p90 {out['gap_us_p90']:.1f}); step span {out['step_span_us_median']:.1f} us")
    print(f"  knn_blocks_kernel {out['knn_us_per_launch_median']:.1f} us x {out['knn_launches_per_step']:.2f}, "
          f"lm_solve_kernel {out['solve_us_per_launch_median']:.1f} us x {out['solve_launches_per_step']:.2f} per step (medians per launch)")
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
