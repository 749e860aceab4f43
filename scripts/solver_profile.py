#!/usr/bin/env python
"""Where the time of one solver launch goes at C2 (bench.py's headline workload: one 100k-pt scan against the 5M-point map).

Runs each distinct scan of bench.make_inputs through scan_to_pose `--reps` times after warm-up and, after every registration, reads the
solver's master-CTA cycle counters (ll_debug_solver_cycles; they cover the last registration).  Prints, per launch (= per ICP iteration):
evaluation, wait, grid reduce, step, staging, epilogue and K10 in microseconds, the evaluations per launch, and the solver's CUDA-event time
(gpu_ms_solve_all / icp_iterations).  Cycles are converted with the SM clock sampled by nvidia-smi (query only) while the registrations run;
the card's name and power limit are read in the same run.  Prints a table and one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

# ll_debug_solver_cycles slots (kernels.cuh: RegDevState::prof); all but [5] are clock64() cycles summed over the last registration
SECTIONS = [("evaluation", 0), ("wait", 1), ("grid_reduce", 2), ("step", 3), ("staging", 6), ("epilogue", 7),
            ("k10_l1_insert", 8), ("k10_select", 10), ("k10_drop", 12), ("compute_step", 13), ("lm_step", 14), ("step_section", 15)]


def gpu_info(device):
    out = subprocess.run(["nvidia-smi", f"--id={device}", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader,nounits"],
                         check=True, capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power, sm = [c.strip() for c in out.split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_mhz_idle_query": float(sm)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20, help="registrations of each distinct scan in the profiled window")
    ap.add_argument("--warmup", type=int, default=3, help="registrations of each distinct scan before the window")
    ap.add_argument("--label", default="", help="tag printed with the results (e.g. which build)")
    args = ap.parse_args()

    import torch
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
    torch.cuda.synchronize()

    def step(k):
        return scan_to_pose(ctx, m, dev_scans[k].data_ptr(), 100.0 + 0.1 * k, pc, states[k], where=capi.LL_DEVICE, n=bench.N_SCAN, fmt=capi.LL_FMT_XYZI16)

    for _ in range(args.warmup):
        for k in range(len(scans)):
            step(k)
    info = gpu_info(device)
    sampler = bench.ClockSampler(device)
    sampler.start()
    cyc_sum = np.zeros(16, np.float64)
    launches, solve_ms = 0, 0.0
    cyc = np.zeros(16, np.int64)
    for _ in range(args.reps):
        for k in range(len(scans)):
            res, _, _ = step(k)
            assert res.status == 1 and res.registered == 1, (k, res.status)
            ctx.check(ctx._lib.ll_debug_solver_cycles(ctx.h, cyc.ctypes.data))
            cyc_sum += cyc
            launches += res.icp_iterations
            solve_ms += res.gpu_ms_solve_all
    clocks = sampler.stop()
    mhz = clocks["sm_mhz"]
    if not mhz:
        raise RuntimeError("no SM clock samples from nvidia-smi: cannot convert cycles to time")

    per_launch_us = {name: cyc_sum[j] / launches / mhz for name, j in SECTIONS}
    evals = cyc_sum[5] / launches
    event_us = 1e3 * solve_ms / launches
    out = {"label": args.label, "gpu": info["name"], "power_limit_w": info["power_limit_w"], "sm_mhz_under_load": mhz, "sm_max_mhz": clocks["sm_max_mhz"],
           "throttle_reasons": clocks["reasons"], "registrations": args.reps * len(scans), "launches": launches,
           "evaluations_per_launch": evals, "solve_event_us_per_launch": event_us, "us_per_launch": per_launch_us,
           "us_per_evaluation": {name: per_launch_us[name] / evals for name in ("evaluation", "wait", "grid_reduce", "step")}}

    print(f"solver profile {args.label}: {info['name']}, power limit {info['power_limit_w']:.0f} W, SM clock {mhz:.0f} MHz under load "
          f"(max {clocks['sm_max_mhz']}, throttle reasons {clocks['reasons'] or 'none'})")
    print(f"  {args.reps * len(scans)} registrations, {launches} launches, {evals:.2f} evaluations per launch, "
          f"CUDA-event solver time {event_us:.1f} us per launch")
    print(f"  {'section':<16}{'us/launch':>11}{'us/eval':>10}")
    for name, _ in SECTIONS:
        per_eval = f"{per_launch_us[name] / evals:10.2f}" if name in out["us_per_evaluation"] else ""
        print(f"  {name:<16}{per_launch_us[name]:11.2f}{per_eval}")
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
