"""Cost of a loop-closure checkpoint (ll_mapper_loop_save / ll_mapper_loop_load; DESIGN.md §4.6.1) on two end states near the reference's scale:

  unclosed: --scans Livox scans of --points points along an out-and-back path, keyframes of 30 scans opened every 10 (the reference's 300 / 100
            ratio) and no candidate search, so every keyframe of the stream is closed and processed and the loop never closes;
  closed:   --closed-scans scans of --closed-points points out along the room, back and out again, keyframes of 6 scans opened every 2 and the
            search of tests/test_gpu_loop_closure.py's parity test, which closes the loop on the return to the start.

Every full cloud goes into the full-resolution cell map, so the full map holds a few million stored points at the defaults.  Before any timing,
each end state is saved (mapper image and loop image), restored on a second context (ll_mapper_load, then ll_mapper_loop_load) and both mappers
run --next more scans: every ll_reg_result field but gpu_ms_*, every integer stat, every loop event, the loop result, the refined clouds and both
end images must be equal, and the restored mapper's loop image saved before those scans must equal the one it was loaded from.  Then, over
--reps repetitions, host wall clock around: save = the size query + the save into a preallocated buffer; load = ll_mapper_loop_load onto a mapper
loaded from the mapper image of the same step, including the loop closure's allocations and the recomputed refined clouds (both end in a device
synchronisation).  The image bytes per second of each and, for comparison, plain pageable host <-> device copies of the same size.  Whether the
loop closed is reported as found, not assumed.  Prints the card and its power limit.

    python scripts/loop_checkpoint.py --scans 60 --points 100000 --closed-scans 90 --closed-points 24000 --reps 5
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from mapper_checkpoint import copy_rate, gpu_info  # noqa: E402

RESERVE = dict(reserve_map_points=1 << 23, reserve_history_points=1 << 22, reserve_keyframes=64)
UNCLOSED = dict(scans_of_each_keyframe=30, scans_between_two_keyframe=10, loop=dict(minimum_keyframe_differen=100000), **RESERVE)
CLOSED = dict(scans_of_each_keyframe=6, scans_between_two_keyframe=2, map_alignment_inlier_threshold=0.35,
              loop=dict(minimum_keyframe_differen=36, avail_ratio_plane=0.02, avail_ratio_line=0.005), **RESERVE)


def returning(n, step=0.15):
    """out along the aisle and back to the start, then out again, n poses"""
    from loam_livox_b200 import synthetic as S
    xs = [0.3 + step * k for k in range(40)] + [0.3 + step * (39 - k) for k in range(40)]
    xs = (xs + xs[1:]) * (1 + n // 80)
    return [S.Pose(np.array([1.0, 0.0, 0.0, 0.0]), np.array([x, 0.2, 0.0])) for x in xs[:n]]


def mapper(ctx, p0):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping
    pipe = capi.PipelineCfg(pieces=3, use_piece=0, extractor_leaf_corner=0.1, extractor_leaf_surf=0.2, mapping_leaf_corner=0.1, mapping_leaf_surf=0.4, whole_frame=1)
    st = capi.default_reg_state(mapping_init_accumulate_frames=3, q_w_last=p0.q, t_w_last=p0.t, q_w_curr=p0.q, t_w_curr=p0.t)
    return Laser_mapping(ctx, reg=st, pipeline=pipe, matching_mode=0, maximum_history_size=400)


def entry(res, st):
    from loam_livox_b200 import capi
    val = lambda x: np.array(list(x) if isinstance(x, C.Array) else [x]).tobytes()  # noqa: E731
    return tuple(val(getattr(res, f)) for f, _ in capi.RegResult._fields_ if not f.startswith("gpu_ms")) + \
        tuple(getattr(st, f) for f, t in capi.MapperStats._fields_ if t is C.c_int)


def event(e):
    """an event's bytes without the pose graph's SM clock counters, which time the solve"""
    from loam_livox_b200 import capi
    c = capi.LoopEvent.from_buffer_copy(e)
    c.summary.cycles_eval = c.summary.cycles_elim = c.summary.cycles_border = c.summary.cycles_total = 0
    return bytes(c)


def run(gm, raws, stamps, chunk=16):
    out = []
    for i in range(0, len(raws), chunk):
        out += [entry(r, s) for r, s in gm.process_new_scans(raws[i:i + chunk], stamps[i:i + chunk])]
    return out


def loop_state(gm):
    r = gm.loop_result()
    clouds = [gm.loop_cloud(k).tobytes() for k in range(r["poses_ori"].shape[0] - 1, -1, -2)] if r["closed"] else []
    return r["closed"], r["poses_ori"].tobytes(), r["poses_opt"].tobytes(), bytes(r["edge"]), clouds


def measure(name, cfg, n, n_pts, n_next, reps):
    from loam_livox_b200 import synthetic as S
    from loam_livox_b200.registration import Context, Laser_mapping, loop_image_info
    poses = returning(n + n_next)
    raws = [S.make_scan(n_pts, p, seed=S.SEED + 7000 + k) for k, p in enumerate(poses)]
    stamps = [100.0 + 0.1 * k for k in range(len(poses))]
    mk = lambda: Context(0, max_scan_points=max(n_pts, 60000), max_features=1 << 20)  # noqa: E731   (max_features: the keyframes' typed clouds)
    a, b = mk(), mk()
    try:
        gm = mapper(a, poses[0])
        gm.set_loop_closure(**cfg)
        t = time.perf_counter()
        run(gm, raws[:n], stamps[:n])
        build_s = time.perf_counter() - t
        mimg, limg = gm.save(), gm.save_loop()
        info = loop_image_info(limg)
        # bit for bit: the saved mapper and its restoration on another context run the next scans alike
        restored = Laser_mapping.load(b, mimg)
        restored.load_loop(limg)
        assert restored.save_loop() == limg, f"{name}: load-then-save differs"
        assert loop_state(restored) == loop_state(gm), f"{name}: the restored loop result or refined clouds differ"
        want, got = run(gm, raws[n:], stamps[n:]), run(restored, raws[n:], stamps[n:])
        assert got == want, f"{name}: the restored mapper parts from the saved one"
        la, lb = gm.loop_log(), restored.loop_log()
        assert [event(e) for e in la[0]] == [event(e) for e in lb[0]] and la[1] == lb[1], f"{name}: the loop events differ"
        assert loop_state(restored) == loop_state(gm) and restored.save() == gm.save() and restored.save_loop() == gm.save_loop(), f"{name}: end states differ"
        restored.close()
        gm.close()
        # timing, on the saved end state: a fresh mapper over the same stream reproduces the image, then save / load repeatedly
        gm = mapper(a, poses[0])
        gm.set_loop_closure(**cfg)
        run(gm, raws[:n], stamps[:n])
        assert gm.save_loop() == limg, f"{name}: the same stream gave another loop image"
        L, n_bytes = a._lib, len(limg)
        buf = np.empty(n_bytes, np.uint8)
        size = C.c_size_t()
        save_s, load_s = [], []
        for _ in range(reps):
            t = time.perf_counter()
            a.check(L.ll_mapper_loop_save(gm.h, None, 0, C.byref(size)))
            a.check(L.ll_mapper_loop_save(gm.h, buf.ctypes.data, n_bytes, C.byref(size)))
            save_s.append(time.perf_counter() - t)
        assert buf.tobytes() == limg
        target = Laser_mapping.load(b, mimg)
        src = np.frombuffer(limg, np.uint8)
        for _ in range(reps):
            t = time.perf_counter()
            b.check(L.ll_mapper_loop_load(target.h, src.ctypes.data, n_bytes, None))
            load_s.append(time.perf_counter() - t)
        target.close()
        gm.close()
        h2d, d2h = copy_rate(n_bytes, reps)
    finally:
        a.close(); b.close()
    save_ms, load_ms = 1e3 * float(np.median(save_s)), 1e3 * float(np.median(load_s))
    return dict(state=name, scans=n, points_per_scan=n_pts, build_s=round(build_s, 1), loop_image_bytes=n_bytes, mapper_image_bytes=len(mimg),
                closed=bool(info["closed"]), keyframes=info["keyframes"], open_keyframes=info["open_keyframes"], cells=info["cells"],
                cell_points=info["cell_points"], replaced_points=info["replaced_points"], history_points=info["history_points"],
                keyframe_cloud_points=info["cloud_points"], accumulated_points=info["accumulated_points"], events=info["events"],
                save_ms=round(save_ms, 2), load_ms=round(load_ms, 2), save_min_ms=round(1e3 * min(save_s), 2), load_min_ms=round(1e3 * min(load_s), 2),
                save_GBps=round(n_bytes / save_ms / 1e6, 2), load_GBps=round(n_bytes / load_ms / 1e6, 2),
                pageable_d2h_GBps=round(d2h / 1e9, 2), pageable_h2d_GBps=round(h2d / 1e9, 2), continuation="bit-identical", next_scans=n_next, reps=reps)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--scans", type=int, default=60, help="scans of the unclosed state")
    ap.add_argument("--points", type=int, default=100000, help="points per scan of the unclosed state")
    ap.add_argument("--closed-scans", type=int, default=90, help="scans of the closed state")
    ap.add_argument("--closed-points", type=int, default=24000, help="points per scan of the closed state")
    ap.add_argument("--next", type=int, default=5, help="scans both mappers run after the restore")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    gpu = gpu_info()
    print(f"card: {gpu['name']}, power limit {gpu['power.limit']}, max SM clock {gpu['clocks.max.sm']}")
    rows = [measure("unclosed", UNCLOSED, args.scans, args.points, args.next, args.reps),
            measure("closed", CLOSED, args.closed_scans, args.closed_points, args.next, args.reps)]
    for r in rows:
        print(f"{r['state']}: {r['scans']} scans of {r['points_per_scan']} points, loop closed {r['closed']}, loop image {r['loop_image_bytes'] / 1e6:.1f} MB "
              f"(keyframes {r['keyframes']} closed / {r['open_keyframes']} open, cells {r['cells']}, kept cell points {r['cell_points']}, "
              f"history {r['history_points']}, keyframe clouds {r['keyframe_cloud_points']}, accumulated {r['accumulated_points']}); "
              f"save {r['save_ms']} ms ({r['save_GBps']} GB/s), load {r['load_ms']} ms ({r['load_GBps']} GB/s); "
              f"pageable copies D2H {r['pageable_d2h_GBps']} GB/s, H2D {r['pageable_h2d_GBps']} GB/s; continuation after restore {r['continuation']}")
    out = dict(gpu=gpu, results=rows)
    print(json.dumps(out))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
