"""The loop image (ll_mapper_loop_save / ll_mapper_loop_load; DESIGN.md §4.6.1): a mapper saved with both images at a cut and restored on a
second context (ll_mapper_load, then ll_mapper_loop_load) continues bit for bit as the saved one, through scans in matching modes 0 and 1,
frames and sweeps: every result and integer stat, every loop event (also across events drained before the save), the loop result, the refined
clouds and, at the end, both images.  Loop images are canonical, and refused images change nothing."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from loam_livox_b200 import synthetic as S  # noqa: E402
from test_gpu_loop_closure import N, SMALL, NOSEARCH, _mapper, _entry, _stats, _ev, _returning, _scans  # noqa: E402

pytestmark = pytest.mark.gpu

LOOP = dict(SMALL, loop=dict(SMALL["loop"], minimum_keyframe_differen=36))   # the parity test's: the return to the start closes the loop


@pytest.fixture(scope="module")
def ctxs():
    from loam_livox_b200.registration import Context
    cs = [Context(0, max_scan_points=60000, max_features=400000) for _ in range(2)]
    yield cs
    for c in cs:
        c.close()


def _restore(ctx, a, **alloc):
    from loam_livox_b200.registration import Laser_mapping
    b = Laser_mapping.load(ctx, a.save())
    b.load_loop(a.save_loop(), **alloc)
    return b


def _same_loop_state(a, b):
    ra, rb = a.loop_result(), b.loop_result()
    assert ra["closed"] == rb["closed"]
    assert ra["poses_ori"].tobytes() == rb["poses_ori"].tobytes() and ra["poses_opt"].tobytes() == rb["poses_opt"].tobytes()
    assert bytes(ra["edge"]) == bytes(rb["edge"])
    if ra["closed"]:
        n = ra["poses_ori"].shape[0]
        for k in range(n - 1, -1, -2):
            assert a.loop_cloud(k).tobytes() == b.loop_cloud(k).tobytes(), k


def _continue_both(a, b, rest):
    """a and b over the same inputs (scans: (raws, stamps)); their entries, stats, events and end states equal."""
    ra, rb = a.process_new_scans(*rest), b.process_new_scans(*rest)
    assert [_entry(x) for x, _ in ra] == [_entry(x) for x, _ in rb]
    assert [_stats(x) for _, x in ra] == [_stats(x) for _, x in rb]


def _finish(a, b, drained):
    """b's log continues a's (a drained `drained` before the save); the loop state and both images are equal."""
    la, da = a.loop_log()
    lb, db = b.loop_log()
    assert da == db
    assert [_ev(e) for e in la] == [_ev(e) for e in lb]
    _same_loop_state(a, b)
    assert a.save() == b.save()
    assert a.save_loop() == b.save_loop()
    return drained + la


# ---------------------------------------------------------------------------------------------- scans: cuts through the stream
def _cut_and_continue(ctxs, mode, poses, raws, stamps, cut, cfg, drain_at=None, **mapper_kw):
    from loam_livox_b200.registration import loop_image_info
    a = _mapper(ctxs[0], mode, poses[0], **mapper_kw)
    a.set_loop_closure(**cfg)
    drained = []
    if drain_at is not None:
        a.process_new_scans(raws[:drain_at], stamps[:drain_at])
        drained = a.loop_log()[0]
        a.process_new_scans(raws[drain_at:cut], stamps[drain_at:cut])
    else:
        a.process_new_scans(raws[:cut], stamps[:cut])
    img = a.save_loop()
    assert a.save_loop() == img   # the save drains nothing
    b = _restore(ctxs[1], a)
    try:
        info = loop_image_info(img)
        _same_loop_state(a, b)
        assert b.save_loop() == img   # load-then-save
        _continue_both(a, b, (raws[cut:], stamps[cut:]))
        log = _finish(a, b, drained)
    finally:
        a.close(); b.close()
    return info, log


@pytest.mark.parametrize("mode", [0, 1])
def test_cuts_before_a_close_with_open_keyframes_and_after_the_loop(ctxs, mode):
    from loam_livox_b200 import capi
    poses = _returning(40) + _returning(40)[1:11]
    raws, stamps = _scans(poses, S.SEED + 5800)
    # keyframes of 6 scans opened every 2: the first closes at step 6; after 3 steps two are open, after 5 three with two accumulated clouds
    info, _ = _cut_and_continue(ctxs, mode, poses, raws, stamps, 3, LOOP)
    assert info["keyframes"] == 0 and info["open_keyframes"] == 2 and not info["closed"]
    info, _ = _cut_and_continue(ctxs, mode, poses, raws, stamps, 5, LOOP)
    assert info["keyframes"] == 0 and info["open_keyframes"] == 3 and info["accumulated_points"] > 0
    # a full run: where the loop closes; then the cut in the step after it, with events drained before the save
    ref = _mapper(ctxs[0], mode, poses[0])
    ref.set_loop_closure(**LOOP)
    out = ref.process_new_scans(raws, stamps)
    log, _ = ref.loop_log()
    closed = [e for e in log if e.kind == capi.LL_LOOP_CLOSED]
    assert closed, "the loop closes on this stream"
    kf = [e for e in log if e.kind == capi.LL_LOOP_KEYFRAME]
    step = [e.ending_frame_idx for e in kf if e.keyframe == closed[0].keyframe][0]   # frame index after the closing step
    want = [_ev(e) for e in log]
    ref_res = ref.loop_result()
    ref.close()
    assert step < len(raws)
    info, got = _cut_and_continue(ctxs, mode, poses, raws, stamps, step, LOOP, drain_at=step - 3)
    assert info["closed"] == 1 and info["keyframes"] >= 2
    assert [_ev(e) for e in got] == want   # drained before the save + read after the load = the uncut run's log
    # mid-stream with events unread across the cut, then the whole log again
    info, got = _cut_and_continue(ctxs, mode, poses, raws, stamps, 30, LOOP)
    assert info["keyframes"] > 0 and info["events"] > 0
    assert [_ev(e) for e in got] == want
    assert len(out) == len(raws) and ref_res["closed"]


def test_a_revisit_held_by_an_open_keyframe_survives_the_image(ctxs):
    """threshold_cell_revisit 4 (as §4.5's end-to-end test): a cell replaced while an open keyframe holds its old incarnation"""
    from loam_livox_b200.registration import loop_image_info
    poses = _returning(20)
    raws, stamps = _scans(poses, S.SEED + 5900)
    a = _mapper(ctxs[0], 0, poses[0], threshold_cell_revisit=4)
    a.set_loop_closure(**NOSEARCH)
    cut = None
    for k in range(len(raws) - 4):
        a.process_new_scans(raws[k:k + 1], stamps[k:k + 1])
        info = loop_image_info(a.save_loop())
        if info["replaced_points"] > 0 and info["max_incarnation"] >= 1:
            cut = k + 1
            break
    assert cut is not None, "no open keyframe held a replaced incarnation"
    b = _restore(ctxs[1], a)
    assert loop_image_info(b.save_loop())["replaced_points"] == info["replaced_points"]
    _continue_both(a, b, (raws[cut:], stamps[cut:]))
    log = _finish(a, b, [])
    from loam_livox_b200 import capi
    assert [e for e in log if e.kind == capi.LL_LOOP_KEYFRAME]
    a.close(); b.close()


# ---------------------------------------------------------------------------------------------- frames and sweeps
def test_a_cut_through_frames(ctxs):
    poses = _returning(12)
    frames = [S.make_triple_scan(N, p, seed=S.SEED + 6000 + 3 * k) for k, p in enumerate(poses)]
    stamps = [[100.0 + 0.1 * k] * 3 for k in range(len(poses))]
    a = _mapper(ctxs[0], 0, poses[0], pieces=2)
    a.set_loop_closure(**NOSEARCH)
    a.process_new_frames(frames[:5], stamps[:5])
    b = _restore(ctxs[1], a)
    ra, rb = a.process_new_frames(frames[5:], stamps[5:]), b.process_new_frames(frames[5:], stamps[5:])
    assert [[_entry(x) for x, _ in f] for f in ra] == [[_entry(x) for x, _ in f] for f in rb]
    assert [[_stats(x) for _, x in f] for f in ra] == [[_stats(x) for _, x in f] for f in rb]
    _finish(a, b, [])
    a.close(); b.close()


def test_a_cut_through_sweeps(ctxs):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_feature, Laser_mapping
    poses = S.trajectory(n_scans=14, n_static=2, speed=1.0)
    raws = [S.make_spinning_scan(16, p, seed=S.SEED + 6100 + k) for k, p in enumerate(poses)]
    fs = [Laser_feature(c, 16) for c in ctxs]
    mk = lambda c: Laser_mapping(c, reg=capi.default_reg_state(mapping_init_accumulate_frames=3, q_w_last=poses[0].q, t_w_last=poses[0].t,
                                                               q_w_curr=poses[0].q, t_w_curr=poses[0].t), matching_mode=0, maximum_history_size=400)
    a = mk(ctxs[0])
    try:
        a.set_loop_closure(**NOSEARCH)
        a.process_new_sweeps(fs[0], raws[:7])
        b = _restore(ctxs[1], a)
        ra, rb = a.process_new_sweeps(fs[0], raws[7:]), b.process_new_sweeps(fs[1], raws[7:])
        assert [_entry(x) for x, _ in ra] == [_entry(x) for x, _ in rb]
        assert [_stats(x) for _, x in ra] == [_stats(x) for _, x in rb]
        log = _finish(a, b, [])
        assert [e for e in log if e.kind == capi.LL_LOOP_KEYFRAME]
        b.close()
    finally:
        a.close()
        for f in fs:
            f.close()


# ---------------------------------------------------------------------------------------------- canonical form
def test_loop_images_are_canonical(ctxs):
    poses = _returning(10)
    raws, stamps = _scans(poses, S.SEED + 6200)
    a, b = _mapper(ctxs[0], 1, poses[0]), _mapper(ctxs[1], 1, poses[0])
    for m in (a, b):
        m.set_loop_closure(**NOSEARCH)
        m.process_new_scans(raws, stamps)
    img = a.save_loop()
    assert b.save_loop() == img   # the same stream on two contexts
    for alloc in ({}, dict(max_cells=1 << 21, reserve_map_points=1 << 16, reserve_history_points=0, reserve_keyframes=3)):
        c = _restore(ctxs[1], a, **alloc)
        assert c.save_loop() == img, alloc   # load-then-save, whatever the allocation sizes
        c.close()
    a.close(); b.close()


# ---------------------------------------------------------------------------------------------- refusals change nothing
def test_refusals_change_nothing(ctxs):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping
    poses = _returning(10)
    raws, stamps = _scans(poses, S.SEED + 6300)
    L = ctxs[0]._lib
    a = _mapper(ctxs[0], 0, poses[0])
    n = C.c_size_t()
    assert L.ll_mapper_loop_save(a.h, None, 0, C.byref(n)) == capi.LL_ERR_INVALID   # loop closure off
    a.set_loop_closure(**NOSEARCH)
    a.process_new_scans(raws[:8], stamps[:8])
    img, mimg = a.save_loop(), a.save()
    # a short cap returns the size and writes nothing
    buf = (C.c_char * (len(img) - 1))()
    assert L.ll_mapper_loop_save(a.h, buf, len(img) - 1, C.byref(n)) == capi.LL_ERR_CAPACITY and n.value == len(img)
    assert bytes(buf) == b"\0" * (len(img) - 1)
    # the target: a restored mapper one step further on, with loop closure of its own
    t = Laser_mapping.load(ctxs[1], mimg)
    t.load_loop(img)
    t.process_new_scans(raws[8:9], stamps[8:9])
    before, limg = t.loop_result(), t.save_loop()

    def unchanged():
        after = t.loop_result()
        assert after["poses_ori"].tobytes() == before["poses_ori"].tobytes() and after["closed"] == before["closed"]
        assert t.save_loop() == limg

    def refused(image, cfg=None, status=capi.LL_ERR_INVALID):
        arr = np.frombuffer(image, np.uint8)
        assert ctxs[1]._lib.ll_mapper_loop_load(t.h, arr.ctypes.data, arr.shape[0], C.byref(cfg) if cfg is not None else None) == status
        unchanged()

    refused(img)   # one step further on: the stamp differs
    # another cell_resolution: in mode 0 the cell maps do not steer the registration, so only that setting differs from the stamp
    other = _mapper(ctxs[1], 0, poses[0], cell_resolution=2.0)
    other.set_loop_closure(**NOSEARCH)
    other.process_new_scans(raws[:8], stamps[:8])
    assert [x.tobytes() if hasattr(x, "tobytes") else x for x in other.pose()] == [x.tobytes() if hasattr(x, "tobytes") else x for x in a.pose()]
    arr = np.frombuffer(img, np.uint8)
    assert ctxs[1]._lib.ll_mapper_loop_load(other.h, arr.ctypes.data, arr.shape[0], None) == capi.LL_ERR_INVALID
    other.close()
    # a config differing outside the allocation fields; too many cells for the effective max_cells (no device work)
    t2 = Laser_mapping.load(ctxs[1], mimg)
    t2.load_loop(img)
    before2, limg2 = t2.loop_result(), t2.save_loop()
    off = int(np.frombuffer(img, np.uint64, count=1, offset=24)[0])
    cfg = capi.LoopClosureCfg.from_buffer_copy(img[off:off + C.sizeof(capi.LoopClosureCfg)])
    bad = capi.LoopClosureCfg.from_buffer_copy(bytes(cfg))
    bad.rng_seed += 1
    assert ctxs[1]._lib.ll_mapper_loop_load(t2.h, arr.ctypes.data, arr.shape[0], C.byref(bad)) == capi.LL_ERR_INVALID
    small = capi.LoopClosureCfg.from_buffer_copy(bytes(cfg))
    small.max_cells = 16
    from loam_livox_b200.registration import loop_image_info
    assert loop_image_info(img)["cells"] > 2048   # more than half of the smallest table (4096 slots)
    assert ctxs[1]._lib.ll_mapper_loop_load(t2.h, arr.ctypes.data, arr.shape[0], C.byref(small)) == capi.LL_ERR_CAPACITY
    after2 = t2.loop_result()
    assert after2["poses_ori"].tobytes() == before2["poses_ori"].tobytes() and t2.save_loop() == limg2
    unchanged()
    a.close(); t.close(); t2.close()
