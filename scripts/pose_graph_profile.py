"""Pose-graph solve on one GPU against the CPU oracle on one thread.

Graphs: a keyframe chain of N poses with drifted odometry (tests/pose_graph_reference.chain_graph) and L loop edges from late keyframes to
early ones, as the reference adds them.  Per graph: the device solve's wall time (host clock around ll_pose_graph_optimize, which returns
after its one synchronising read-back; median of --reps after one warm-up), its LM iterations, the time per iteration, the split of the
kernel's cycles between evaluation, segment elimination and the border system, and the oracle's wall time on one CPU thread.

    python scripts/pose_graph_profile.py [--sizes 300 3000 30000 100000] [--loops 1 32] [--reps 5] [--json out.json]
"""
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

import pose_graph_reference as R  # noqa: E402
from loam_livox_b200.registration import Context, PoseGraph, pg_edges  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e})"


def graph(n, loops, seed):
    rng = np.random.default_rng(seed)
    truth = R.trajectory(n, rng)
    lp = [(int(n - 1 - k * max(1, n // 200)), int(rng.integers(0, n // 4))) for k in range(loops)]
    return R.chain_graph(truth, rng, lp)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[300, 3000, 30000, 100000])
    ap.add_argument("--loops", type=int, nargs="+", default=[1, 32])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-max", type=int, default=100000, help="largest graph the oracle is timed on")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    info = gpu_info()
    import torch
    clock_khz = torch.cuda.get_device_properties(0).clock_rate if hasattr(torch.cuda.get_device_properties(0), "clock_rate") else None
    print(f"GPU: {info}")
    ctx = Context(0, max_scan_points=1000, max_features=1000)
    pg = PoseGraph(ctx, max(a.sizes), max(a.sizes) + max(a.loops))
    R.oracle_lib()   # compiled once here, outside the timed calls
    rows = []
    for n in a.sizes:
        for L in a.loops:
            X, ids, meas = graph(n, L, n + L)
            E = pg_edges(ids[:, 0], ids[:, 1], meas[:, :4], meas[:, 4:7])
            pg.optimize(X, E)
            ts = []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                xd, s = pg.optimize(X, E)
                ts.append(time.perf_counter() - t0)
            ms = 1e3 * float(np.median(ts))
            cyc = np.array([s.cycles_eval, s.cycles_elim, s.cycles_border, s.cycles_total], np.float64)
            row = dict(n=n, loops=L, gpu_ms=ms, iterations=s.iterations, evaluations=s.evaluations, termination=s.termination,
                       ms_per_iteration=ms / max(1, s.iterations), border=s.border_nodes, segments=s.segments, levels=s.levels,
                       cycle_share_eval=cyc[0] / cyc[3], cycle_share_elim=cyc[1] / cyc[3], cycle_share_border=cyc[2] / cyc[3])
            if clock_khz:
                row["kernel_ms_at_max_clock"] = cyc[3] / clock_khz
            if n <= a.oracle_max:
                t0 = time.perf_counter()
                xo, c0, c1, it, ev, term = R.oracle_optimize(X, ids, meas)
                row["oracle_ms"] = 1e3 * (time.perf_counter() - t0)
                row["oracle_iterations"] = it
                row["max_dt_vs_oracle"] = float(np.abs(xd[:, 4:] - xo[:, 4:]).max())
            rows.append(row)
            print(json.dumps(row))
    pg.close()
    ctx.close()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(gpu=info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
