#!/usr/bin/env python
"""Where the front end of a C2 step goes (bench.py's headline workload: one 100k-pt scan through ll_scan_to_pose against the 5M-point map).

Two runs over the distinct scans of bench.make_inputs, after warm-up:
  timing:   CUDA events around each step on the context's stream (the L2 flushed before it, as bench.py does) minus the registration's own
            gpu_ms_total: the front end (extraction, get_features, the four VoxelGrids) plus its count read-back and the host gap behind it;
  profiler: torch.profiler (CUDA activity only), one profiled window per step.  The kernels that run before the registration's first kernel
            (the query sort's key kernel) are the front end's: a kernel table per step, the front end's span (first kernel start to last
            front-end kernel end) and the VoxelGrid chains' span (first VoxelGrid kernel start to last VoxelGrid kernel end).
The card's name and power limit are read in the same run.  Prints a table and one JSON line.

    python scripts/front_end_profile.py --steps 60 --label parent
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from solver_profile import gpu_info  # noqa: E402

REGISTRATION_FIRST = ("query_key_kernel", "knn_blocks")   # the first kernel of register_device's work
VOXEL_GRID = ("vg_", "DeviceRadixSort", "DeviceSelect", "DeviceScan", "Onesweep", "onesweep")


def is_vg(name):
    return any(t in name for t in VOXEL_GRID) and "ex_" not in name


def short(name, width=72):
    name = name.replace("void ", "")
    return name if len(name) <= width else name[:width - 3] + "..."


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60, help="timed steps (cycling through the distinct scans); the profiled run takes a third of them")
    ap.add_argument("--warmup", type=int, default=3, help="steps of each distinct scan before each run")
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
    torch.cuda.synchronize()

    def step(k):
        return scan_to_pose(ctx, m, dev_scans[k].data_ptr(), 100.0 + 0.1 * k, pc, states[k], where=capi.LL_DEVICE, n=bench.N_SCAN, fmt=capi.LL_FMT_XYZI16)

    def warm():
        for _ in range(args.warmup):
            for k in range(nd):
                step(k)
        torch.cuda.synchronize()

    info = gpu_info(device)
    # ---- timing run
    warm()
    sampler = bench.ClockSampler(device)
    sampler.start()
    step_ms, reg_ms = [], []
    for i in range(args.steps):
        with torch.cuda.stream(stream):
            flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        res, _, _ = step(i % nd)
        b.record(stream)
        b.synchronize()
        assert res.status == 1 and res.registered == 1, (i, res.status)
        step_ms.append(a.elapsed_time(b))
        reg_ms.append(res.gpu_ms_total)
    clocks = sampler.stop()
    step_ms, reg_ms = np.array(step_ms), np.array(reg_ms)
    front_ms = step_ms - reg_ms

    # ---- profiler run (separate: tracing slows the host)
    warm()
    table, fe_span, vg_span, fe_kernel_sum, vg_kernel_sum = {}, [], [], [], []
    n_prof = max(1, args.steps // 3)
    for i in range(n_prof):
        with torch.cuda.stream(stream):
            flush.zero_()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step(i % nd)
            torch.cuda.synchronize()
        ks = sorted([(e.time_range.start, e.time_range.end, e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                     and e.time_range.end > e.time_range.start and "Memcpy" not in e.name and "Memset" not in e.name and "elementwise" not in e.name
                     and "fill" not in e.name.lower()])
        first_reg = next((t0 for t0, _, n in ks if any(r in n for r in REGISTRATION_FIRST)), None)
        assert first_reg is not None, "no registration kernel found in the trace"
        fe = [k for k in ks if k[0] < first_reg]
        vg = [k for k in fe if is_vg(k[2])]
        fe_span.append(max(e for _, e, _ in fe) - fe[0][0])
        vg_span.append((max(e for _, e, _ in vg) - vg[0][0]) if vg else 0.0)
        fe_kernel_sum.append(sum(e - s for s, e, _ in fe))
        vg_kernel_sum.append(sum(e - s for s, e, _ in vg))
        for s, e, n in fe:
            t = table.setdefault(short(n), [0, 0.0])
            t[0] += 1; t[1] += e - s

    out = {"label": args.label, "gpu": info["name"], "power_limit_w": info["power_limit_w"], "sm_mhz_under_load": clocks["sm_mhz"],
           "throttle_reasons": clocks["reasons"], "steps": args.steps, "profiled_steps": n_prof,
           "step_ms_median": float(np.median(step_ms)), "registration_ms_median": float(np.median(reg_ms)),
           "front_end_plus_readback_ms_median": float(np.median(front_ms)), "front_end_plus_readback_ms_mean": float(np.mean(front_ms)),
           "profiled": {"front_end_span_us_median": float(np.median(fe_span)), "voxel_grid_span_us_median": float(np.median(vg_span)),
                        "front_end_kernel_us_per_step": float(np.mean(fe_kernel_sum)), "voxel_grid_kernel_us_per_step": float(np.mean(vg_kernel_sum)),
                        "kernels_per_step": {k: {"launches": c / n_prof, "us": t / n_prof} for k, (c, t) in sorted(table.items(), key=lambda kv: -kv[1][1])}}}
    print(f"front end profile {args.label}: {info['name']}, power limit {info['power_limit_w']:.0f} W, SM clock {clocks['sm_mhz']} MHz under load "
          f"(throttle reasons {clocks['reasons'] or 'none'})")
    print(f"  step {out['step_ms_median']:.3f} ms, registration {out['registration_ms_median']:.3f} ms, front end + read-back {out['front_end_plus_readback_ms_median']:.3f} ms (medians of {args.steps})")
    p = out["profiled"]
    print(f"  profiled ({n_prof} steps): front-end span {p['front_end_span_us_median']:.1f} us, VoxelGrid span {p['voxel_grid_span_us_median']:.1f} us, "
          f"kernel time {p['front_end_kernel_us_per_step']:.1f} us (VoxelGrid {p['voxel_grid_kernel_us_per_step']:.1f} us)")
    print(f"  {'kernel':<74}{'launches':>9}{'us':>9}")
    for k, v in p["kernels_per_step"].items():
        print(f"  {k:<74}{v['launches']:9.2f}{v['us']:9.1f}")
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
