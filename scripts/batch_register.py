"""B independent registrations against one map, three ways: B serial ll_register calls on one context, B contexts on B host threads (as
bench.py --contexts B), and one ll_register_batch call.  On the C2 workload of bench.py (100k-point scans, 5M-point map, the bench's pipeline
leaves), once with the precision defaults of the benchmark and once under the shipped residual-block cap of 200.

Every item is a C2 scan (6 distinct scans, as bench.py makes them) with its own initial guess; the features come from the library's front end.
Before anything is timed, every output of every arm is checked against the oracle's registration of that item (status, ICP iterations, pose
within 1e-6: at this size the single call itself is 1.1e-7 rad from the oracle under the cap of 200) and the arms against each other (one
context per thread = serial calls bit for bit, the batch within 1e-9).  Prints the card, its power limit and one JSON line per (config, B).

    python scripts/batch_register.py [--sizes 2 4 8 16] [--reps 30]

A batch whose items' slots do not fit the shared memory of their CTA groups (LL_ERR_CAPACITY) is reported as such, with no batch number.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from loam_livox_b200 import capi, synthetic as S  # noqa: E402
from loam_livox_b200.registration import Context, Livox_laser, LoamLivoxError, Map, register_batch, voxel_grid_filter  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi unavailable)"


def features(ctx, raw):
    lx = Livox_laser(ctx)
    lx.extract_laser_features(raw, 100.0)
    c, s, _ = lx.get_features(0.0, 1.0)
    P = bench.PIPE
    c = voxel_grid_filter(ctx, voxel_grid_filter(ctx, c, P["extractor_leaf_corner"]), P["mapping_leaf_corner"])
    s = voxel_grid_filter(ctx, voxel_grid_filter(ctx, s, P["extractor_leaf_surf"]), P["mapping_leaf_surf"])
    return c, s


def single(ctx, m, item, state):
    c, s = item
    res = capi.RegResult()
    ctx.check(ctx._lib.ll_register(ctx.h, m.h, c.ctypes.data, c.shape[0], s.ctypes.data, s.shape[0], capi.LL_FMT_XYZI16, capi.LL_HOST, C.byref(state), C.byref(res)))
    return res


def pose_err(a, b):
    return float(np.linalg.norm(np.array(a.t_w_curr) - np.array(b.t_w_curr))), float(S.quat_angle(np.array(a.q_w_curr), np.array(b.q_w_curr)))


def pose_diff(a, b):
    """Largest component difference of two poses (quat_angle's acos resolves nothing below ~1.5e-8)."""
    return max(np.abs(np.array(a.t_w_curr) - np.array(b.t_w_curr)).max(), np.abs(np.array(a.q_w_curr) - np.array(b.q_w_curr)).max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[2, 4, 8, 16])
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    from oracle import oracle as O
    B_max = max(args.sizes)
    mc, ms, scans, guesses, truths = bench.make_inputs(0, "c2")
    ctxs = [Context(0, max_scan_points=bench.N_SCAN, max_features=bench.N_SCAN * (B_max if k == 0 else 1)) for k in range(B_max)]
    m = Map(ctxs[0], mc, ms)
    feats = [features(ctxs[0], raw) for raw in scans]
    rng = np.random.default_rng(S.SEED + 77)
    items, item_guess = [], []
    for k in range(B_max):   # item k: scan k mod 6; the first 6 start from bench.py's guesses, the rest from fresh perturbations of the truth
        items.append(feats[k % len(scans)])
        item_guess.append(guesses[k] if k < len(scans) else S.perturb_pose(truths[k % len(scans)], rng))
    trees = (O.KdTree(mc), O.KdTree(ms))
    print(f"card: {card()}", flush=True)
    print(f"features per scan: {[a.shape[0] + b.shape[0] for a, b in feats]}", flush=True)
    for cfg_name, extra in (("c2", {}), ("c2_cap200", dict(maximum_allow_residual_block=200, max_final_cost=2.0))):
        states = [capi.default_reg_state(q_w_last=g.q, t_w_last=g.t, q_w_curr=g.q, t_w_curr=g.t, rng_seed=k, **extra) for k, g in enumerate(item_guess)]
        # ---- outputs first: every item through the oracle, the serial arm, the threaded arm and the batch arm
        oracle_res = []
        for k in range(B_max):
            g = item_guess[k]
            p = O.default_params(q_w_last=g.q, t_w_last=g.t, q_w_curr=g.q, t_w_curr=g.t, rng_seed=k, num_threads=bench.host_threads(), **extra)
            oracle_res.append(O.register(mc, trees[0], ms, trees[1], items[k][0], items[k][1], p))
        worst, fits = 0.0, {}
        for B in args.sizes:
            serial = [single(ctxs[0], m, items[k], states[k]) for k in range(B)]
            threaded = [None] * B
            def work(k):
                threaded[k] = single(ctxs[k], m, items[k], states[k])
            ths = [threading.Thread(target=work, args=(k,)) for k in range(B)]
            [t.start() for t in ths]; [t.join() for t in ths]
            try:
                batch, status = register_batch(ctxs[0], m, items[:B], states[:B])
                assert status == [capi.LL_OK] * B, status
                fits[B] = True
            except LoamLivoxError as e:   # the items' slots do not fit the shared memory of their CTA groups
                assert "status -3" in str(e), e
                print(f"{cfg_name} B={B}: the batch does not fit ({e})", flush=True)
                fits[B], batch = False, serial
            for k in range(B):
                ost, ores = oracle_res[k]
                for arm, r in (("serial", serial[k]), ("threads", threaded[k]), ("batch", batch[k])):
                    dt, da = pose_err(r, ores)
                    assert r.status == ost and r.icp_iterations == ores.icp_iterations and dt < 1e-6 and da < 1e-6, (cfg_name, B, k, arm, r.status, ost, dt, da)
                    worst = max(worst, dt, da)
                assert pose_diff(serial[k], threaded[k]) == 0.0 and pose_diff(serial[k], batch[k]) <= 1e-9
        print(f"{cfg_name}: every output of every arm agrees with the oracle (largest pose deviation {worst:.1e})", flush=True)
        # ---- timing (host clock around calls that end in a device synchronise)
        for B in args.sizes:
            def run_serial():
                for k in range(B):
                    single(ctxs[0], m, items[k], states[k])
            def run_threads():
                ths = [threading.Thread(target=lambda k=k: single(ctxs[k], m, items[k], states[k])) for k in range(B)]
                [t.start() for t in ths]; [t.join() for t in ths]
            def run_batch():
                register_batch(ctxs[0], m, items[:B], states[:B])
            line = {"config": cfg_name, "B": B, "reps": args.reps, "card": card()}
            for name, fn in (("serial", run_serial), ("threads", run_threads), ("batch", run_batch)):
                if name == "batch" and not fits[B]:
                    line["batch_scans_per_s"] = None
                    continue
                for _ in range(2):
                    fn()
                t0 = time.perf_counter()
                for _ in range(args.reps):
                    fn()
                dt = time.perf_counter() - t0
                line[f"{name}_scans_per_s"] = round(B * args.reps / dt, 1)
            print(json.dumps(line), flush=True)
    for c in ctxs:
        c.close()


if __name__ == "__main__":
    main()
