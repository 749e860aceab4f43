"""Checkpoint and resume of the streaming mapper (ll_mapper_save / ll_mapper_load): a mapper saved after any input and restored on another,
fresh context continues exactly as the uninterrupted one -- every ll_reg_result field but the gpu_ms_* timings bit for bit, every integer
field of ll_mapper_stats, the pose and the frame index -- on every front-end path; saving changes nothing; images are canonical; the
image's counts equal the oracle's; refused images create nothing."""
import ctypes as C
import os
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from loam_livox_b200 import synthetic as S  # noqa: E402

N = 24000


def _capi():
    from loam_livox_b200 import capi
    return capi


def entry(res, st):
    capi = _capi()
    val = lambda x: np.array(list(x) if isinstance(x, C.Array) else [x]).tobytes()  # noqa: E731
    return tuple(val(getattr(res, f)) for f, _ in capi.RegResult._fields_ if not f.startswith("gpu_ms")) + \
        tuple(getattr(st, f) for f, t in capi.MapperStats._fields_ if t is C.c_int)


def state(gm):
    q, t, f = gm.pose()
    return q.tobytes(), t.tobytes(), f


def new_ctx(device=0):
    from loam_livox_b200.registration import Context
    return Context(device, max_scan_points=60000, max_features=60000)


def mapper(ctx, pieces=3, mode=0, window=3, init=3, **kw):
    from loam_livox_b200.registration import Laser_mapping
    capi = _capi()
    reg = {k: kw.pop(k) for k in list(kw) if hasattr(capi.RegState, k)}
    pipe = capi.PipelineCfg(pieces=pieces, use_piece=0, extractor_leaf_corner=0.1, extractor_leaf_surf=0.2, mapping_leaf_corner=0.1, mapping_leaf_surf=0.4, whole_frame=1)
    return Laser_mapping(ctx, reg=capi.default_reg_state(mapping_init_accumulate_frames=init, **reg), pipeline=pipe, matching_mode=mode, maximum_history_size=window, **kw)


def scans(n, seed):
    poses = S.trajectory(n_scans=n, n_static=2, speed=1.0)
    return [S.make_scan(N, p, seed=seed + k) for k, p in enumerate(poses)], [100.0 + 0.1 * k for k in range(n)]


def frames(n, seed, heads=1):
    poses = S.trajectory(n_scans=n, n_static=2, speed=1.0)
    if heads == 1:
        return [[S.make_scan(N, p, seed=seed + k)] for k, p in enumerate(poses)], [[100.0 + 0.1 * k] for k in range(n)]
    return [S.make_triple_scan(3 * 16000, p, seed=seed + 3 * k) for k, p in enumerate(poses)], [[100.0 + 0.1 * k] * 3 for k in range(n)]


def scan_steps(raws, stamps):
    return lambda gm, i: [entry(*gm.process_new_scan(raws[i], stamps[i]))]


def frame_steps(fr, stamps, odom_mode=1):
    return lambda gm, i: [entry(r, s) for r, s in gm.process_new_frame(fr[i], stamps[i], odom_mode)]


def section(img, k):
    off, length = struct.unpack_from("<QQ", img, 24 + 16 * k)
    return img[off:off + length]


def history_sizes(img, c):
    h = section(img, _capi().LL_IMAGE_HISTORY_CORNER + c)
    n_seg, _ = struct.unpack_from("<qq", h, 0)
    return list(struct.unpack_from(f"<{n_seg}i", h, 16))


def run_with_saves(make, step, n, ctx, at=None):
    """(entries, end state, {k: image after k inputs}) of one run that saves after the inputs in `at` (every one by default)."""
    gm = make(ctx)
    at = set(range(n + 1)) if at is None else set(at)
    images, out = {}, []
    if 0 in at:
        images[0] = gm.save()
    for i in range(n):
        out.append(step(gm, i))
        if i + 1 in at:
            images[i + 1] = gm.save()
    st = state(gm)
    gm.close()
    return out, st, images


def check_resume(make, step, n, at=None, alloc=None, rest=None):
    """The uninterrupted run (no saves) on one context; the same run saving after the inputs in `at` on another (equal: saving changes
    nothing; the final images of both equal: canonical); every image restored on a fresh context (alloc: buffer sizes of the new mapper) and
    run to the end (by `rest`, default the single calls) equal to the uninterrupted run, its image reproduced by a save right after the
    load.  Returns (entries, images)."""
    from loam_livox_b200.registration import Laser_mapping
    a, b = new_ctx(), new_ctx()
    try:
        ref = make(a)
        want = [step(ref, i) for i in range(n)]
        final, final_image = state(ref), ref.save()
        ref.close()
        got, st, images = run_with_saves(make, step, n, b, at)
        assert got == want and st == final
        if n in images:
            assert images[n] == final_image
    finally:
        a.close(); b.close()
    for k, img in sorted(images.items()):
        other = new_ctx()
        try:
            gm = Laser_mapping.load(other, img, **(alloc(images) if alloc else {}))
            assert gm.save() == img, k
            cont = rest(gm, k) if rest else [step(gm, i) for i in range(k, n)]
            assert cont == want[k:], k
            assert state(gm) == final, k
            gm.close()
        finally:
            other.close()
    return want, images


def small_table(images):
    """max_cells just above the largest cell map any image of the stream holds (the run's end state has the most cells), reservations 0."""
    from loam_livox_b200.registration import image_info
    cells = max(max(image_info(img)["cells"]) for img in images.values())
    return dict(max_cells=cells + 1, reserve_map_points=0, reserve_store_points=0)


# ---------------------------------------------------------------------------------------------- resume anywhere
@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("override", [False, True])
def test_resume_after_every_scan(mode, override):
    """8 scans, a window of 3 clouds that pops, the init gate crossed at scan 3: saved after every k = 0 ... 8 and resumed on a fresh
    context.  override: a much smaller table and no reservations, so slot layout and buffer sizes differ from the saved mapper's."""
    from loam_livox_b200.registration import image_info
    raws, stamps = scans(8, S.SEED + 5000 + 100 * mode)
    want, images = check_resume(lambda c: mapper(c, mode=mode), scan_steps(raws, stamps), 8, alloc=small_table if override else None)
    assert any(e[0][1] == np.array([1]).tobytes() for e in want)   # some scan registered
    fresh = image_info(images[0])
    assert fresh["frame_index"] == 0 and fresh["cells"] == [0, 0] and fresh["history_segments"] == [0, 0] and fresh["have_map"] == 0
    last = image_info(images[8])
    assert last["frame_index"] == 8 and last["history_segments"] == [3, 3] and last["have_map"] == 1 and min(last["cell_points"]) > 0


# ---------------------------------------------------------------------------------------------- every front-end path
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["pieces3", "heads3", "deblur", "sequences"])
def test_resume_on_every_front_end_path(name):
    if name == "sequences":   # restored, then the sequence calls: process_new_frames, then process_new_scans
        fr, st = frames(6, S.SEED + 5300)
        raws, ts = scans(4, S.SEED + 5400)
        ts = [101.0 + 0.1 * k for k in range(4)]

        def step(gm, i):
            return frame_steps(fr, st)(gm, i) if i < 6 else scan_steps(raws, ts)(gm, i - 6)

        def rest(gm, k):
            out = [[entry(r, s) for r, s in f] for f in gm.process_new_frames(fr[k:], st[k:])] if k < 6 else []
            return out + [[entry(r, s)] for r, s in gm.process_new_scans(raws[max(k - 6, 0):], ts[max(k - 6, 0):])]
        check_resume(lambda c: mapper(c, mode=1), step, 10, at=[0, 2, 6, 8], rest=rest)
        return
    kw, heads = {"pieces3": (dict(), 1), "heads3": (dict(pieces=2), 3), "deblur": (dict(init=2, if_motion_deblur=1), 1)}[name]
    fr, st = frames(6, S.SEED + 5500, heads)
    want, _ = check_resume(lambda c: mapper(c, **kw), frame_steps(fr, st), 6, at=[1, 2, 4])
    assert sum(len(f) for f in want) == 6 * (1 if name == "deblur" else kw.get("pieces", 3))


# ---------------------------------------------------------------------------------------------- state that is easy to miss
@pytest.mark.gpu
def test_resume_after_a_rejected_registration():
    """A tight max_final_cost rejects registrations: a save right after one holds a clean match map (map_dirty 0), whose snapshot and index
    the next step uses as they are."""
    from loam_livox_b200.registration import image_info
    raws, stamps = scans(7, S.SEED + 5600)
    want, images = check_resume(lambda c: mapper(c, mode=1, max_final_cost=1e-7), scan_steps(raws, stamps), 7)
    rejected = [k + 1 for k, e in enumerate(want) if e[0][0] == np.array([0]).tobytes()]
    assert rejected
    for k in rejected:
        info = image_info(images[k])
        assert info["map_dirty"] == 0 and info["have_map"] == 1


@pytest.mark.gpu
@pytest.mark.parametrize("replace", [0, 1])
def test_resume_with_dead_points(replace):
    """Mode 1 with threshold_cell_revisit = 2: revisited cells leave dead points in the store.  Without down-sample-and-replace the store holds
    every point ever appended, and the image's live points are fewer; with it, the dead points of an append live until the next refresh."""
    from loam_livox_b200.registration import image_info
    raws, stamps = scans(8, S.SEED + 5700)
    make = lambda c: mapper(c, mode=1, threshold_cell_revisit=2, down_sample_replace=replace)  # noqa: E731
    want, images = check_resume(make, scan_steps(raws, stamps), 8)
    if not replace:
        capi = _capi()
        n_res = len([f for f, _ in capi.RegResult._fields_ if not f.startswith("gpu_ms")])   # an entry: the result fields, then the integer stats
        ints = [f for f, t in capi.MapperStats._fields_ if t is C.c_int]
        stored = [sum(e[0][n_res + ints.index(f)] for e in want) for f in ("appended_corner", "appended_surf")]
        live = image_info(images[8])["cell_points"]
        assert live[0] < stored[0] or live[1] < stored[1], (live, stored)


# ---------------------------------------------------------------------------------------------- against the oracle
@pytest.mark.gpu
def test_image_counts_equal_the_oracle(oracle):
    """The same mode-1 stream on the device mapper and oracle.Mapper: per cell map the cell count, live points and frame index, and the
    history window's segment sizes, equal the oracle's."""
    from loam_livox_b200.registration import Context, Laser_mapping, image_info
    capi = _capi()
    poses = S.trajectory(n_scans=9, n_static=4, speed=1.0)
    ctx = Context(0, max_scan_points=60000, max_features=60000)
    try:
        gm = Laser_mapping(ctx, reg=capi.default_reg_state(mapping_init_accumulate_frames=3), matching_mode=1, maximum_history_size=3)
        om = oracle.Mapper(oracle.default_params(mapping_init_accumulate_frames=3, num_threads=4), threads=4, matching_mode=1, maximum_history_size=3)
        for k, pose in enumerate(poses):
            raw = S.make_scan(N, pose, seed=S.SEED + k)
            res, _ = gm.process_new_scan(raw, 100.0 + 0.1 * k)
            assert res.status == om.process_scan(raw, 100.0 + 0.1 * k)[0]
            img = gm.save()
            info = image_info(img)
            for c, (cells, his) in enumerate(((om.cells_corner, om.his_corner), (om.cells_surf, om.his_surf))):
                assert (info["cells"][c], info["cell_points"][c], info["cell_frame_idx"][c]) == (cells.cells(), cells.points(), cells.frame_idx()), (k, c)
                assert history_sizes(img, c) == [h.shape[0] for h in his], (k, c)
            assert info["frame_index"] == om.frame_index
        gm.close()
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------- refusals on a live context
def corrupt(img):
    """(name, corrupted image, expected status) of a real image."""
    capi = _capi()
    b = bytes(img)

    def at(k, off, fmt, value):
        o, _ = struct.unpack_from("<QQ", b, 24 + 16 * k)
        x = bytearray(b)
        struct.pack_into(fmt, x, o + off, value)
        return bytes(x)
    mm = capi.MapperConfig.matching_mode.offset
    cells = capi.LL_IMAGE_CELLS_SURF
    n_cells = struct.unpack_from("<q", section(b, cells), 8)[0]
    out = [("truncated", b[:-1], capi.LL_ERR_INVALID), ("magic", b"X" + b[1:], capi.LL_ERR_INVALID),
           ("version", b[:8] + struct.pack("<I", 9) + b[12:], capi.LL_ERR_INVALID), ("config_bytes", b[:12] + struct.pack("<I", 8) + b[16:], capi.LL_ERR_INVALID),
           ("overlap", b[:24 + 16 * 3] + struct.pack("<Q", struct.unpack_from("<Q", b, 24 + 16 * 2)[0]) + b[24 + 16 * 3 + 8:], capi.LL_ERR_INVALID),
           ("matching_mode", at(capi.LL_IMAGE_CONFIG, mm, "<i", 2), capi.LL_ERR_INVALID),
           ("pose", at(capi.LL_IMAGE_SCALARS, 40, "<d", float("nan")), capi.LL_ERR_INVALID),
           ("key_bit63", at(cells, 24 + 7, "<B", 0x80), capi.LL_ERR_INVALID),
           ("rank", at(cells, 24 + 16 * n_cells + 12, "<i", n_cells), capi.LL_ERR_INVALID),
           ("stamp", at(cells, 24 + 8, "<i", 1 << 30), capi.LL_ERR_INVALID),
           ("history_count", at(capi.LL_IMAGE_HISTORY_CORNER, 0, "<q", 99), capi.LL_ERR_INVALID)]
    return out


@pytest.mark.gpu
def test_refused_images_create_nothing():
    """Each corrupted image returns its status on a live context and creates no mapper; a table too small for the image's cells is
    LL_ERR_CAPACITY.  A mapper then created on that context runs a stream equal to one on a fresh context.  Cells of 0.05 m, so that the
    image holds more cells than the smallest table (4096 slots) takes."""
    from loam_livox_b200.registration import image_config, image_info
    capi = _capi()
    raws, stamps = scans(8, S.SEED + 5800)
    step = scan_steps(raws, stamps)
    make = lambda c: mapper(c, mode=1, cell_resolution=0.1)  # noqa: E731
    ctx = new_ctx()
    try:
        gm = make(ctx)
        for i in range(6):
            step(gm, i)
        img = gm.save()
        gm.close()
        L = ctx._lib

        def load(image, cfg=None):
            h, buf = C.c_void_p(), np.frombuffer(image, np.uint8)
            st = L.ll_mapper_load(ctx.h, buf.ctypes.data, buf.shape[0], C.byref(cfg) if cfg is not None else None, C.byref(h))
            if h.value:
                L.ll_mapper_release(h)
            return st, h.value
        for name, bad, code in corrupt(img):
            assert load(bad) == (code, None), name
        assert max(image_info(img)["cells"]) > 2048
        cfg = image_config(img)
        cfg.max_cells = 16
        assert load(img, cfg) == (capi.LL_ERR_CAPACITY, None)
        cfg = image_config(img)
        cfg.line_resolution = 0.2   # not a buffer size
        assert load(img, cfg) == (capi.LL_ERR_INVALID, None)
        gm = make(ctx)
        got = [step(gm, i) for i in range(8)]
        gm.close()
    finally:
        ctx.close()
    fresh = new_ctx()
    try:
        gm = make(fresh)
        assert [step(gm, i) for i in range(8)] == got
        gm.close()
    finally:
        fresh.close()


# ---------------------------------------------------------------------------------------------- another GPU
@pytest.mark.gpu
def test_resume_on_another_gpu():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    from loam_livox_b200.registration import Laser_mapping
    raws, stamps = scans(6, S.SEED + 5900)
    step = scan_steps(raws, stamps)
    a = new_ctx(0)
    try:
        gm = mapper(a, mode=1)
        want = [step(gm, i) for i in range(6)]
        final = state(gm)
        gm.close()
        gm = mapper(a, mode=1)
        for i in range(3):
            step(gm, i)
        img = gm.save()
        gm.close()
    finally:
        a.close()
    b = new_ctx(1)
    try:
        gm = Laser_mapping.load(b, img)
        assert [step(gm, i) for i in range(3, 6)] == want[3:] and state(gm) == final
        gm.close()
    finally:
        b.close()
