"""Spinning-lidar front end (ll_spin_extract) on VLP-16- and HDL-64-sized sweeps in the room and in an open scene: device time per scan
(CUDA events around the call, after warm-up), kernel launches per call, the selection's chains and the longest one, the oracle's time on one
CPU thread, and the card's name and power limit, read in the same run.  One JSON line per workload, then a summary line."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from loam_livox_b200 import synthetic as S  # noqa: E402
from loam_livox_b200.registration import Context, Laser_feature  # noqa: E402
from oracle.spin_oracle import SpinExtractor  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    import torch
    ctx = Context(0, max_scan_points=1000, max_features=1000)
    fronts = {16: Laser_feature(ctx, 16), 64: Laser_feature(ctx, 64)}
    stream = torch.cuda.ExternalStream(ctx.stream())
    rows = []
    for scan_line, n_az in ((16, 1800), (64, 2080)):
        for scene in ("room", "open"):
            raw = S.make_spinning_scan(scan_line, n_azimuth=n_az, scene=scene, seed=1, nan_frac=0.01, start_azimuth_deg=30.0)
            f = fronts[scan_line]
            for _ in range(a.warmup):
                f.extract(raw)
            l0 = ctx.launches()
            f.extract(raw)
            launches = ctx.launches() - l0
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record(stream)
            for _ in range(a.iters):
                f.extract(raw)
            ev[1].record(stream)
            ev[1].synchronize()
            ms = ev[0].elapsed_time(ev[1]) / a.iters
            chains, longest = f.chains()
            o = SpinExtractor(scan_line)
            o.extract(raw)
            row = dict(scan_line=scan_line, scene=scene, points=int(raw.shape[0]), counts=[int(c) for c in f.counts], ms_per_scan=round(ms, 4),
                       launches_per_call=int(launches), chains=chains, longest_chain_points=longest, oracle_ms_one_thread=round(o.seconds * 1e3, 3))
            rows.append(row)
            print(json.dumps(row))
    print(json.dumps({"card": card(), "iters": a.iters, "warmup": a.warmup, "note": "host-input calls: upload, extract and the count read-back"}))
    for f in fronts.values():
        f.close()
    ctx.close()


if __name__ == "__main__":
    main()
