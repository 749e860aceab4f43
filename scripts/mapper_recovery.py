"""Cost of the streaming mapper's tracking-loss recovery (ll_mapper_set_recovery; DESIGN.md §4.3.2) on one GPU:

  idle:    process_new_scans scans/s on a C3-style stream (24k-point scans, matching mode 0) with recovery off and with recovery on under the
           defaults (idle: no step is bad).  The two arms' outputs (results, integer stats, pose, mapper image) are compared first; then the arms
           alternate over --reps repetitions, each on a fresh mapper of its own context.
  kidnap:  the stream of tests/test_gpu_recovery.py (the sensor moved 1 m back, 2 m aside and turned 15 deg at scan 160) in both matching modes:
           per attempt the host milliseconds of the map + field build and of the search, the steps lost and the error of every later pose
           from the synthetic truth.

The card, its power limit and SM clock are read in the same call.  --out PATH also writes the measurements to PATH as JSON.

    python scripts/mapper_recovery.py --scans 200 --reps 5
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


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.splitlines()[0].split(",")]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import test_gpu_recovery as T
    from loam_livox_b200 import synthetic as S
    from loam_livox_b200.registration import Context
    info = gpu_info()
    print(f"card: {info['name']}, power limit {info['power.limit']}, SM clock {info['clocks.sm']} (max {info['clocks.max.sm']})")
    ctx = [Context(0, max_scan_points=60000, max_features=60000) for _ in range(2)]
    poses, raws, stamps = T._stream(a.scans, S.SEED + 3100)

    def run(arm, c):
        lm = T._mapper(c, 0, poses[0])
        if arm == "idle":
            lm.set_recovery()
        c.sync()
        t0 = time.perf_counter()
        rs = lm.process_new_scans(raws, stamps)
        dt = time.perf_counter() - t0
        return lm, rs, dt

    # outputs first
    la, ra, _ = run("off", ctx[0])
    lb, rb, _ = run("idle", ctx[1])
    assert [T._entry(x) for x, _ in ra] == [T._entry(x) for x, _ in rb] and [T._stats(x) for _, x in ra] == [T._stats(x) for _, x in rb]
    assert la.save() == lb.save() and all(e.bad == 0 for e in lb.recovery_log()[0])
    la.close(); lb.close()
    rate = {"off": [], "idle": []}
    for r in range(a.reps):
        for arm in (("off", "idle") if r % 2 == 0 else ("idle", "off")):
            lm, _, dt = run(arm, ctx[0 if arm == "off" else 1])
            rate[arm].append(a.scans / dt)
            lm.close()
    for arm, v in rate.items():
        print(f"{arm:5s} scans/s: median {np.median(v):.1f}, min {min(v):.1f}, max {max(v):.1f} over {len(v)} runs")
    # the kidnap stream
    n = T.K_JUMP + 12
    kp, kr, ks = T._stream(n, S.SEED + 2300, jump=T.K_JUMP)
    kid = {}
    for mode in (0, 1):
        lm = T._mapper(ctx[0], mode, kp[0])
        lm.set_recovery()
        rs = lm.process_new_scans(kr, ks)
        log, _ = lm.recovery_log()
        att = [e for e in log if e.attempted]
        adopted = [k for k, e in enumerate(log) if e.adopted]
        errs = [T._err(np.array(r.q_w_curr), np.array(r.t_w_curr), kp[k]) for k, (r, _) in enumerate(rs)][adopted[0] + 1:] if adopted else []
        kid[mode] = {"attempts": [{"frame": e.frame_index, "ms_map": e.ms_map, "ms_search": e.ms_search, "n_cand": e.n_cand, "best": e.best,
                                   "verify_fraction": e.verify_fraction, "adopted": e.adopted, "grew": e.grew, "nt": list(e.nt)} for e in att],
                     "steps_lost": (adopted[0] - T.K_JUMP + 1) if adopted else None,
                     "max_err_after": [max(x[0] for x in errs), max(x[1] for x in errs)] if errs else None}
        print(f"kidnap mode {mode}: {json.dumps(kid[mode])}")
        lm.close()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        json.dump({"gpu": info, "scans_per_s": rate, "kidnap": kid}, open(a.out, "w"), indent=1)
    for c in ctx:
        c.close()


if __name__ == "__main__":
    main()
