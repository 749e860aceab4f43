"""Cost of a mapper checkpoint (ll_mapper_save / ll_mapper_load) on two end states:

  c3:    a C3-style stream (matching_mode 0, window 400, 100k-point scans, the leaves of bench.py --workload c3) run until the mode-0 cell
         store (which only grows) holds a few million points;
  mode1: the same scans in matching_mode 1 (cells in range and in the FOV, down-sample-and-replace).

Before any timing, every end state is saved, restored on a second context and both mappers run the next scans: their results must be equal
(every ll_reg_result field but gpu_ms_*, every integer field of the stats, the pose), and the restored mapper's image must equal the saved one.
Then, over --reps repetitions, host wall clock around: save = the size query + the save into a preallocated buffer; load = ll_mapper_load,
including the index rebuild (both end in a device synchronisation).  The image bytes per second of each, and, for comparison, a plain
pageable host <-> device copy of the same size (the transfers inside save and load are such copies).  Prints the card and its power limit.

    python scripts/mapper_checkpoint.py --scans 300 --mode1-scans 150 --reps 5
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_PTS, INIT, WINDOW, LINE, PLANE, NEXT = 100000, 50, 400, 0.05, 0.1, 5


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.splitlines()[0].split(",")]))


def mapper(ctx, mode):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping
    pipe = capi.PipelineCfg(pieces=3, use_piece=0, extractor_leaf_corner=LINE, extractor_leaf_surf=PLANE / 2, mapping_leaf_corner=LINE, mapping_leaf_surf=PLANE, whole_frame=1)
    return Laser_mapping(ctx, reg=capi.default_reg_state(mapping_init_accumulate_frames=INIT), pipeline=pipe, line_resolution=LINE, plane_resolution=PLANE,
                         matching_mode=mode, maximum_history_size=WINDOW, reserve_map_points=1 << 22, reserve_store_points=1 << 23)


def key(res, st):
    from loam_livox_b200 import capi
    val = lambda x: np.array(list(x) if isinstance(x, C.Array) else [x]).tobytes()  # noqa: E731
    return tuple(val(getattr(res, f)) for f, _ in capi.RegResult._fields_ if not f.startswith("gpu_ms")) + \
        tuple(getattr(st, f) for f, t in capi.MapperStats._fields_ if t is C.c_int)


def scans(n):
    from loam_livox_b200 import synthetic as S
    poses = S.trajectory(n_scans=n, n_static=INIT + 1, speed=1.0, zero_mean_yaw=True, y0=-1.6)
    return [S.make_scan(N_PTS, poses[k], seed=S.SEED + k) for k in range(n)], [100.0 + 0.1 * k for k in range(n)]


def run(gm, raws, stamps, chunk=32):
    out = []
    for i in range(0, len(raws), chunk):
        out += [key(r, s) for r, s in gm.process_new_scans(raws[i:i + chunk], stamps[i:i + chunk])]
    return out


def copy_rate(n_bytes, reps):
    """Bytes/s of a pageable host -> device and device -> host copy of n_bytes (torch, synchronised), median over reps."""
    import torch
    host = torch.from_numpy(np.ones(n_bytes, np.uint8))
    dev = torch.empty(n_bytes, dtype=torch.uint8, device="cuda")
    h2d, d2h = [], []
    for _ in range(reps):
        torch.cuda.synchronize(); t = time.perf_counter(); dev.copy_(host); torch.cuda.synchronize(); h2d.append(time.perf_counter() - t)
        t = time.perf_counter(); host.copy_(dev); torch.cuda.synchronize(); d2h.append(time.perf_counter() - t)
    return n_bytes / float(np.median(h2d)), n_bytes / float(np.median(d2h))


def measure(name, mode, n, reps):
    from loam_livox_b200.registration import Context, Laser_mapping, image_info
    raws, stamps = scans(n + NEXT)
    a, b = Context(0, max_scan_points=N_PTS, max_features=N_PTS), Context(0, max_scan_points=N_PTS, max_features=N_PTS)
    try:
        gm = mapper(a, mode)
        t = time.perf_counter()
        run(gm, raws[:n], stamps[:n])
        build_s = time.perf_counter() - t
        image = gm.save()
        info = image_info(image)
        # bit for bit: the saved mapper and its restoration on another context run the next scans alike
        restored = Laser_mapping.load(b, image)
        assert restored.save() == image, f"{name}: load-then-save differs"
        want, got = run(gm, raws[n:], stamps[n:]), run(restored, raws[n:], stamps[n:])
        assert got == want and [x.tobytes() for x in gm.pose()[:2]] == [x.tobytes() for x in restored.pose()[:2]], f"{name}: the restored mapper parts from the saved one"
        restored.close()
        gm.close()
        gm = mapper(a, mode)
        run(gm, raws[:n], stamps[:n])
        assert gm.save() == image, f"{name}: the same stream gave another image"
        L, n_bytes = a._lib, len(image)
        buf = np.empty(n_bytes, np.uint8)
        size = C.c_size_t()
        save_s, load_s = [], []
        for _ in range(reps):
            t = time.perf_counter()
            a.check(L.ll_mapper_save(gm.h, None, 0, C.byref(size)))
            a.check(L.ll_mapper_save(gm.h, buf.ctypes.data, n_bytes, C.byref(size)))
            save_s.append(time.perf_counter() - t)
        assert buf.tobytes() == image
        src = np.frombuffer(image, np.uint8)
        for _ in range(reps):
            h = C.c_void_p()
            t = time.perf_counter()
            b.check(L.ll_mapper_load(b.h, src.ctypes.data, n_bytes, None, C.byref(h)))
            load_s.append(time.perf_counter() - t)
            L.ll_mapper_release(h)
        gm.close()
        h2d, d2h = copy_rate(n_bytes, reps)
    finally:
        a.close(); b.close()
    save_ms, load_ms = 1e3 * float(np.median(save_s)), 1e3 * float(np.median(load_s))
    return dict(stream=name, matching_mode=mode, scans=n, build_s=round(build_s, 1), image_bytes=n_bytes, cells=info["cells"], cell_points=info["cell_points"],
                history_points=info["history_points"], snapshot_points=info["snapshot_points"], save_ms=round(save_ms, 2), load_ms=round(load_ms, 2),
                save_min_ms=round(1e3 * min(save_s), 2), load_min_ms=round(1e3 * min(load_s), 2),
                save_GBps=round(n_bytes / save_ms / 1e6, 2), load_GBps=round(n_bytes / load_ms / 1e6, 2),
                pageable_d2h_GBps=round(d2h / 1e9, 2), pageable_h2d_GBps=round(h2d / 1e9, 2), continuation="bit-identical", reps=reps)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--scans", type=int, default=300, help="scans of the mode-0 (C3-style) stream")
    ap.add_argument("--mode1-scans", type=int, default=150, help="scans of the mode-1 stream")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    gpu = gpu_info()
    print(f"card: {gpu['name']}, power limit {gpu['power.limit']}, max SM clock {gpu['clocks.max.sm']}")
    rows = [measure("c3", 0, args.scans, args.reps), measure("mode1", 1, args.mode1_scans, args.reps)]
    for r in rows:
        print(f"{r['stream']}: {r['scans']} scans, image {r['image_bytes'] / 1e6:.1f} MB (cells {r['cells']}, live cell points {r['cell_points']}, "
              f"history {r['history_points']}, snapshot {r['snapshot_points']}); save {r['save_ms']} ms ({r['save_GBps']} GB/s), "
              f"load {r['load_ms']} ms ({r['load_GBps']} GB/s); pageable copies D2H {r['pageable_d2h_GBps']} GB/s, H2D {r['pageable_h2d_GBps']} GB/s; "
              f"continuation after restore {r['continuation']}")
    out = dict(gpu=gpu, results=rows)
    print(json.dumps(out))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
