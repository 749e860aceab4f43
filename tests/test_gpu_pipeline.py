"""The sequence calls of the streaming mapper (ll_mapper_process_frames / _scans: the front end of input k + 1 runs on the device while input k
is registered) against the same inputs run one by one (ll_mapper_process_frame / _scan, the same loop over one input with nothing enqueued
ahead) on a mapper and context of their own: every ll_reg_result field but the gpu_ms_* timings bit for bit, every integer field of
ll_mapper_stats, the pose, the frame index and the kernel launch count.  Also the error paths: validation before anything is enqueued, and a
piece or scan over max_features in mid-sequence."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from loam_livox_b200 import synthetic as S  # noqa: E402

N = 24000


def _capi():
    from loam_livox_b200 import capi
    return capi


def _res_fields():
    return [n for n, _ in _capi().RegResult._fields_ if not n.startswith("gpu_ms")]


def _stat_fields():
    return [n for n, t in _capi().MapperStats._fields_ if t is C.c_int]


def entry(res, st):
    """What must be identical between the two arms: every non-timing field of the result, every integer field of the stats."""
    val = lambda x: np.array(list(x) if isinstance(x, C.Array) else [x]).tobytes()  # noqa: E731
    return tuple(val(getattr(res, f)) for f in _res_fields()) + tuple(getattr(st, f) for f in _stat_fields())


def state(gm):
    q, t, f = gm.pose()
    return q.tobytes(), t.tobytes(), f


@pytest.fixture(scope="module")
def ctxs():
    from loam_livox_b200.registration import Context
    a, b = Context(0, max_scan_points=60000, max_features=60000), Context(0, max_scan_points=60000, max_features=60000)
    yield a, b
    a.close(); b.close()


def pipeline(pieces=3, whole_frame=1):
    return _capi().PipelineCfg(pieces=pieces, use_piece=0, extractor_leaf_corner=0.1, extractor_leaf_surf=0.2, mapping_leaf_corner=0.1, mapping_leaf_surf=0.4,
                               whole_frame=whole_frame)


def mapper(ctx, pieces=3, mode=0, window=3, init=3, whole_frame=1, max_cells=0, **reg):
    from loam_livox_b200.registration import Laser_mapping
    return Laser_mapping(ctx, reg=_capi().default_reg_state(mapping_init_accumulate_frames=init, **reg), pipeline=pipeline(pieces, whole_frame),
                         matching_mode=mode, maximum_history_size=window, max_cells=max_cells)


def frames_single(gm, frames, stamps, odom_mode=1):
    return [[entry(r, s) for r, s in gm.process_new_frame(h, t, odom_mode)] for h, t in zip(frames, stamps)]


def frames_seq(gm, frames, stamps, odom_mode=1, split=None, **kw):
    out, i = [], 0
    for n in split or [len(frames)]:
        out += [[entry(r, s) for r, s in f] for f in gm.process_new_frames(frames[i:i + n], stamps[i:i + n], odom_mode, **kw)]
        i += n
    return out


def scans_single(gm, raws, stamps):
    return [entry(*gm.process_new_scan(r, t)) for r, t in zip(raws, stamps)]


def scans_seq(gm, raws, stamps, split=None, **kw):
    out, i = [], 0
    for n in split or [len(raws)]:
        out += [entry(r, s) for r, s in gm.process_new_scans(raws[i:i + n], stamps[i:i + n], **kw)]
        i += n
    return out


def run_pair(ctxs, make, single, seq):
    """(one-by-one entries, sequence entries) on fresh mappers, each on its own context, with equal launch counts and end states."""
    ga, gb = make(ctxs[0]), make(ctxs[1])
    la, lb = ctxs[0].launches(), ctxs[1].launches()
    want, got = single(ga), seq(gb)
    assert ctxs[0].launches() - la == ctxs[1].launches() - lb
    assert state(ga) == state(gb)
    ga.close(); gb.close()
    return want, got


def stream_frames(n, seed, heads=1):
    poses = S.trajectory(n_scans=n, n_static=2, speed=1.0)
    if heads == 1:
        return [[S.make_scan(N, p, seed=seed + k)] for k, p in enumerate(poses)], [[100.0 + 0.1 * k] for k in range(n)]
    return [S.make_triple_scan(3 * 16000, p, seed=seed + 3 * k) for k, p in enumerate(poses)], [[100.0 + 0.1 * k] * 3 for k in range(n)]


# ---------------------------------------------------------------------------------------------- frames
@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1])
def test_frames_match_one_by_one_in_every_split(ctxs, mode):
    """8 frames x 3 pieces, odom_mode 1, a window of 3 clouds that pops, the init gate crossed in frame 1: calls of 1, 2, 7 + 1 and all 8 frames
    each give the one-by-one results; two runs of the same sequence are bit-identical."""
    frames, stamps = stream_frames(8, S.SEED + 2000)
    make = lambda c: mapper(c, mode=mode)  # noqa: E731
    want = None
    for split in ([1] * 8, [2] * 4, [7, 1], [8], [8]):
        w, got = run_pair(ctxs, make, lambda g: frames_single(g, frames, stamps), lambda g: frames_seq(g, frames, stamps, split=split))
        assert got == w, split
        assert want is None or w == want
        want = w
    assert sum(len(f) for f in want) == 24 and any(e[1] == np.array([1]).tobytes() for f in want for e in f)   # some piece registered


def _case(name, oracle):
    """(mapper kwargs, frames, stamps, odom_mode) of one frame-stream case."""
    if name == "odom_mode_0":
        f, t = stream_frames(5, S.SEED + 2100)
        return dict(), f, t, 0
    if name == "deblur":
        f, t = stream_frames(6, S.SEED + 2200)
        return dict(pieces=3, init=2, if_motion_deblur=1), f, t, 1
    if name == "mid100_dropped_heads":
        f, t = stream_frames(6, S.SEED + 2300, heads=3)
        f[3][1] = f[3][1][: f[3][1].shape[0] // 8]   # one head of <= 5 petals
        f[4] = [h[:200] for h in f[4]]               # no head contributes
        return dict(pieces=2), f, t, 1
    if name == "overlapping_16":
        from test_gpu_pieces import few_petals
        poses = S.trajectory(n_scans=3, n_static=2, speed=1.0)
        f = [[few_petals(S.make_scan(N, p, seed=S.SEED + 2400 + k), oracle, 6 + k)] for k, p in enumerate(poses)]
        return dict(pieces=16, init=100), f, [[100.0 + 0.1 * k] for k in range(3)], 1
    if name == "rejected_piece":
        f, t = stream_frames(4, S.SEED + 2500)
        return dict(max_final_cost=1e-7), f, t, 1
    raise KeyError(name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["odom_mode_0", "deblur", "mid100_dropped_heads", "overlapping_16", "rejected_piece"])
def test_frame_cases_match_one_by_one(ctxs, oracle, name):
    kw, frames, stamps, odom = _case(name, oracle)
    want, got = run_pair(ctxs, lambda c: mapper(c, **kw), lambda g: frames_single(g, frames, stamps, odom), lambda g: frames_seq(g, frames, stamps, odom))
    assert got == want
    if name == "mid100_dropped_heads":
        assert want[4] == [] and len(want[3]) == 2
    if name == "rejected_piece":
        assert any(e[0] == np.array([0]).tobytes() for f in want for e in f)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["track_m0_w400", "track_m0_w3", "track_m1_w400", "track_heads3_p2"])
def test_golden_pieces_through_process_frames(ctxs, name):
    """tests/golden/golden_pieces.npz through one process_new_frames call: bit-identical to the one-by-one arm, and within the bars the
    one-by-one test holds it to (counts and ICP iterations exactly, pose 1e-6)."""
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    import make_golden_pieces as G
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "golden_pieces.npz"))[name]
    heads3 = name == "track_heads3_p2"
    mode, window = (0, 400) if heads3 else (int(name[7]), int(name.split("_w")[1]))
    frames = G.head_frames() if heads3 else G.frames()
    stamps = [G.stamps(k, len(h)) for k, h in enumerate(frames)]
    make = lambda c: mapper(c, pieces=G.HEADS_PIECES if heads3 else G.PIECES, mode=mode, window=window, init=G.INIT)  # noqa: E731
    gb = make(ctxs[1])
    out = gb.process_new_frames(frames, stamps)
    rows = [[r.status, 0, s.n_corner, s.n_surf, s.map_corner, s.map_surf, s.appended_corner, s.appended_surf, r.icp_iterations if r.registered else 0]
            + list(r.q_w_curr) + list(r.t_w_curr) for f in out for r, s in f]
    got = np.array(rows)
    assert got.shape == gold.shape
    assert np.array_equal(got[:, [0, 2, 3, 4, 5, 6, 7, 8]], gold[:, [0, 2, 3, 4, 5, 6, 7, 8]])
    assert np.abs(got[:, 9:] - gold[:, 9:]).max() < 1e-6
    assert gb.pose()[2] == int(gold[-1, 1])
    ga = make(ctxs[0])
    assert frames_single(ga, frames, stamps) == [[entry(r, s) for r, s in f] for f in out] and state(ga) == state(gb)
    ga.close(); gb.close()


# ---------------------------------------------------------------------------------------------- scans
@pytest.mark.gpu
@pytest.mark.parametrize("mode,window", [(0, 400), (0, 3), (1, 400)])
def test_golden_stream_through_process_scans(ctxs, mode, window):
    """tests/golden/golden_stream.npz through one process_new_scans call: bit-identical to the one-by-one arm, and within the golden bars."""
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    import make_golden_stream as G
    from loam_livox_b200.registration import Laser_mapping
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "golden_stream.npz"))[f"track_m{mode}_w{window}"]
    raws = G.scans()
    stamps = [100.0 + 0.1 * k for k in range(len(raws))]
    make = lambda c: Laser_mapping(c, reg=_capi().default_reg_state(mapping_init_accumulate_frames=G.INIT), matching_mode=mode, maximum_history_size=window)  # noqa: E731
    gb = make(ctxs[1])
    out = gb.process_new_scans(raws, stamps)
    for k, (res, st) in enumerate(out):
        w = gold[k]
        assert (res.status, st.n_corner, st.n_surf, st.map_corner, st.map_surf, st.appended_corner, st.appended_surf) == tuple(int(x) for x in w[[0, 2, 3, 4, 5, 6, 7]]), k
        assert (res.icp_iterations if res.registered else 0) == int(w[8]), k
    q, t, f = gb.pose()
    assert f == int(gold[-1, 1]) and np.linalg.norm(t - gold[-1, 13:16]) < 1e-6 and S.quat_angle(q, gold[-1, 9:13]) < 1e-6
    ga = make(ctxs[0])
    assert scans_single(ga, raws, stamps) == [entry(r, s) for r, s in out] and state(ga) == state(gb)
    ga.close(); gb.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("whole_frame", [1, 0])
def test_scans_match_one_by_one(ctxs, mode, whole_frame):
    """10 scans in calls of 3 + 7 and of 10; with whole_frame 0 two scans of <= 5 petals are dropped."""
    poses = S.trajectory(n_scans=10, n_static=2, speed=1.0)
    raws = [S.make_scan(N, p, seed=S.SEED + 2600 + k) for k, p in enumerate(poses)]
    if not whole_frame:
        raws[3], raws[6] = raws[3][:200].copy(), raws[6][:300].copy()
    stamps = [100.0 + 0.1 * k for k in range(10)]
    make = lambda c: mapper(c, mode=mode, whole_frame=whole_frame)  # noqa: E731
    for split in ([3, 7], [10]):
        want, got = run_pair(ctxs, make, lambda g: scans_single(g, raws, stamps), lambda g: scans_seq(g, raws, stamps, split=split))
        assert got == want, split
    if not whole_frame:
        assert want[3][_res_fields().index("registered")] == np.array([0]).tobytes()   # dropped: nothing registered


# ---------------------------------------------------------------------------------------------- formats
def _single_raw_scan(gm, ptr, n, fmt, where, stamp):
    capi = _capi()
    res, st = capi.RegResult(), capi.MapperStats()
    gm.ctx.check(gm.ctx._lib.ll_mapper_process_scan(gm.h, C.c_void_p(ptr), n, fmt, where, stamp, C.byref(res), C.byref(st)))
    return entry(res, st)


def _strided(raw, step=20):
    """PointCloud2-style records: x y z at 0 / 4 / 8, a pad, float intensity at 16."""
    rec = np.zeros((raw.shape[0], step), np.uint8)
    rec[:, 0:12] = raw[:, :3].astype(np.float32).view(np.uint8).reshape(-1, 12)
    rec[:, 16:20] = raw[:, 3:4].astype(np.float32).view(np.uint8).reshape(-1, 4)
    return rec


@pytest.mark.gpu
def test_formats_and_device_inputs(ctxs):
    """LL_FMT_PCL32 frames, LL_FMT_STRIDED scans and device-resident inputs of both calls give the one-by-one results."""
    import torch
    capi = _capi()
    frames, stamps = stream_frames(4, S.SEED + 2700)
    pcl = [[np.concatenate([h[:, :3], np.zeros((h.shape[0], 1), np.float32), h[:, 3:4], np.zeros((h.shape[0], 3), np.float32)], axis=1) for h in f] for f in frames]
    want, got = run_pair(ctxs, mapper, lambda g: frames_single(g, pcl, stamps), lambda g: frames_seq(g, pcl, stamps))
    assert got == want and want == run_pair(ctxs, mapper, lambda g: frames_single(g, frames, stamps), lambda g: frames_single(g, frames, stamps))[0]
    dev = [[torch.from_numpy(h).cuda() for h in f] for f in frames]
    torch.cuda.synchronize()
    _, got = run_pair(ctxs, mapper, lambda g: frames_single(g, frames, stamps),
                      lambda g: frames_seq(g, [[h.data_ptr() for h in f] for f in dev], stamps, where=capi.LL_DEVICE, ns=[[h.shape[0] for h in f] for f in dev],
                                           fmt=capi.LL_FMT_XYZI16))
    assert got == want
    raws = [f[0] for f in frames]
    ts = [t[0] for t in stamps]
    recs = [_strided(r) for r in raws]
    for c in ctxs:
        c.set_point_layout(20, 0, 4, 8, 16, capi.LL_I_FLOAT32)
    try:
        want, got = run_pair(ctxs, mapper, lambda g: [_single_raw_scan(g, r.ctypes.data, r.shape[0], capi.LL_FMT_STRIDED, capi.LL_HOST, t) for r, t in zip(recs, ts)],
                             lambda g: scans_seq(g, recs, ts, fmt=capi.LL_FMT_STRIDED, ns=[r.shape[0] for r in recs]))
        assert got == want and want == run_pair(ctxs, mapper, lambda g: scans_single(g, raws, ts), lambda g: scans_single(g, raws, ts))[0]
    finally:
        for c in ctxs:
            c.set_point_layout(16)
    dev = [torch.from_numpy(r).cuda() for r in raws]
    torch.cuda.synchronize()
    _, got = run_pair(ctxs, mapper, lambda g: scans_single(g, raws, ts),
                      lambda g: scans_seq(g, [d.data_ptr() for d in dev], ts, where=capi.LL_DEVICE, ns=[d.shape[0] for d in dev], fmt=capi.LL_FMT_XYZI16))
    assert got == want


# ---------------------------------------------------------------------------------------------- mixing and errors
@pytest.mark.gpu
def test_sequences_interleave_with_single_calls(ctxs):
    """On one mapper: frames in calls of 2, 1 (single), 3, 1 (single), 1; then scans in calls of 1 (single), 3, 1 (single), 2 -- the one-by-one
    results throughout."""
    frames, stamps = stream_frames(8, S.SEED + 2800)
    poses = S.trajectory(n_scans=7, n_static=0, speed=1.0)
    raws = [S.make_scan(N, p, seed=S.SEED + 2900 + k) for k, p in enumerate(poses)]
    ts = [101.0 + 0.1 * k for k in range(7)]

    def mixed(g):
        out, i = [], 0
        for n, single in ((2, False), (1, True), (3, False), (1, True), (1, False)):
            out += frames_single(g, frames[i:i + n], stamps[i:i + n]) if single else frames_seq(g, frames[i:i + n], stamps[i:i + n])
            i += n
        i = 0
        for n, single in ((1, True), (3, False), (1, True), (2, False)):
            out += scans_single(g, raws[i:i + n], ts[i:i + n]) if single else scans_seq(g, raws[i:i + n], ts[i:i + n])
            i += n
        return out
    want, got = run_pair(ctxs, mapper, lambda g: frames_single(g, frames, stamps) + scans_single(g, raws, ts), mixed)
    assert got == want


def _frames_call(gm, frames, stamps, odom_mode=1, cap=16, n_frames=None, n_heads=None, fmt=None, where=None, ns=None, null=None):
    """ll_mapper_process_frames directly: (status, *n_frames_done, n_pieces, entries of the completed pieces)."""
    capi = _capi()
    nf, nh = len(frames), len(frames[0])
    arrs = [np.ascontiguousarray(h, np.float32) for f in frames for h in f]
    ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
    if null is not None:
        ptrs[null] = None
    sizes = (C.c_size_t * len(arrs))(*(ns or [a.shape[0] for a in arrs]))
    st = (C.c_double * len(arrs))(*[t for f in stamps for t in f])
    res, stats = (capi.RegResult * (nf * max(cap, 1)))(), (capi.MapperStats * (nf * max(cap, 1)))()
    n_pieces, done = (C.c_int * nf)(*([-1] * nf)), C.c_int(-1)
    status = gm.ctx._lib.ll_mapper_process_frames(gm.h, nf if n_frames is None else n_frames, nh if n_heads is None else n_heads, ptrs, sizes,
                                                  capi.LL_FMT_XYZI16 if fmt is None else fmt, capi.LL_HOST if where is None else where, st, odom_mode, res, stats, cap,
                                                  n_pieces, C.byref(done))
    ok = max(done.value, 0)
    entries = [[entry(res[f * cap + i], stats[f * cap + i]) for i in range(n_pieces[f])] for f in range(min(ok + 1, nf)) if n_pieces[f] >= 0]
    return status, done.value, list(n_pieces), entries


def _scans_call(gm, raws, stamps, n_scans=None, fmt=None, where=None, ns=None, null=None):
    capi = _capi()
    arrs = [np.ascontiguousarray(r, np.float32) for r in raws]
    ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
    if null is not None:
        ptrs[null] = None
    sizes = (C.c_size_t * len(arrs))(*(ns or [a.shape[0] for a in arrs]))
    st = (C.c_double * len(arrs))(*stamps)
    res, stats, done = (capi.RegResult * len(arrs))(), (capi.MapperStats * len(arrs))(), C.c_int(-1)
    status = gm.ctx._lib.ll_mapper_process_scans(gm.h, len(arrs) if n_scans is None else n_scans, ptrs, sizes, capi.LL_FMT_XYZI16 if fmt is None else fmt,
                                                 capi.LL_HOST if where is None else where, st, res, stats, C.byref(done))
    return status, done.value, [entry(res[k], stats[k]) for k in range(max(done.value, 0))]


@pytest.mark.gpu
def test_validation_errors_change_nothing(ctxs):
    """Every validation error of the sequence and the single calls returns before anything is enqueued: nothing done, pose and frame index
    unchanged, and the next call continues exactly as the one-by-one arm.  After a rejected single call the mapper's image (which holds the
    extractor's time bookkeeping) is that of a mapper that never saw the call, also when the call was the first input of a fresh mapper."""
    capi = _capi()
    frames, stamps = stream_frames(5, S.SEED + 3000)
    raws, ts = [f[0] for f in frames], [t[0] for t in stamps]
    ga, gb = mapper(ctxs[0]), mapper(ctxs[1])
    want = frames_single(ga, frames[:2], stamps[:2])
    assert frames_seq(gb, frames[:2], stamps[:2]) == want
    before = state(gb)
    big = ctxs[1].cfg.max_scan_points + 1
    two, st2 = frames[2:4], stamps[2:4]
    for kw, code in ((dict(n_frames=0), capi.LL_ERR_INVALID), (dict(n_heads=0), capi.LL_ERR_INVALID), (dict(n_heads=9), capi.LL_ERR_INVALID),
                     (dict(odom_mode=2), capi.LL_ERR_INVALID), (dict(cap=2), capi.LL_ERR_INVALID), (dict(fmt=7), capi.LL_ERR_INVALID),
                     (dict(where=5), capi.LL_ERR_INVALID), (dict(null=1), capi.LL_ERR_INVALID), (dict(ns=[N, big]), capi.LL_ERR_CAPACITY)):
        status, done, n_pieces, _ = _frames_call(gb, two, st2, **kw)
        assert status == code and done == 0 and state(gb) == before, kw
    for kw, code in ((dict(n_scans=0), capi.LL_ERR_INVALID), (dict(fmt=7), capi.LL_ERR_INVALID), (dict(where=5), capi.LL_ERR_INVALID),
                     (dict(null=1), capi.LL_ERR_INVALID), (dict(ns=[N, big]), capi.LL_ERR_CAPACITY)):
        status, done, _ = _scans_call(gb, raws[2:4], ts[2:4], **kw)
        assert status == code and done == 0 and state(gb) == before, kw
    assert frames_seq(gb, frames[2:], stamps[2:]) == frames_single(ga, frames[2:], stamps[2:]) and state(ga) == state(gb)
    ga.close(); gb.close()
    # the single calls: gb sees each rejected call, then both take the next input; the first case is the first input of a fresh mapper,
    # stamped apart from the first real input
    frames, stamps = stream_frames(6, S.SEED + 3050)
    raws, ts = [f[0] for f in frames], [t[0] for t in stamps]
    cases = ((dict(fmt=7, stamps=[50.0]), capi.LL_ERR_INVALID), (dict(where=5), capi.LL_ERR_INVALID), (dict(null=0), capi.LL_ERR_INVALID),
             (dict(ns=[big]), capi.LL_ERR_CAPACITY), (dict(odom_mode=2), capi.LL_ERR_INVALID), (dict(cap=2), capi.LL_ERR_INVALID))
    ga, gb = mapper(ctxs[0]), mapper(ctxs[1])
    for k, (kw, code) in enumerate(cases):
        assert _raw_frame(gb, frames[k], **{"stamps": stamps[k], **kw}) == (code, 0, []), kw
        assert state(gb) == state(ga) and gb.save() == ga.save(), kw
        assert frames_single(gb, frames[k:k + 1], stamps[k:k + 1]) == frames_single(ga, frames[k:k + 1], stamps[k:k + 1]), kw
    assert state(gb) == state(ga) and gb.save() == ga.save()
    ga.close(); gb.close()
    cases = ((dict(fmt=7, stamp=50.0), capi.LL_ERR_INVALID), (dict(where=5), capi.LL_ERR_INVALID), (dict(null=True), capi.LL_ERR_INVALID),
             (dict(n=big), capi.LL_ERR_CAPACITY))
    ga, gb = mapper(ctxs[0]), mapper(ctxs[1])
    for k, (kw, code) in enumerate(cases):
        assert _single_raw_scan_status(gb, raws[k], **{"stamp": ts[k], **kw})[0] == code, kw
        assert state(gb) == state(ga) and gb.save() == ga.save(), kw
        assert scans_single(gb, raws[k:k + 1], ts[k:k + 1]) == scans_single(ga, raws[k:k + 1], ts[k:k + 1]), kw
    assert state(gb) == state(ga) and gb.save() == ga.save()
    ga.close(); gb.close()


@pytest.mark.gpu
def test_max_features_in_mid_sequence(ctxs):
    """A frame with a piece over max_features in the middle of a sequence stops it there: LL_ERR_CAPACITY, the frames before it and the pieces
    of it completed as the one-by-one arm that hit the same error; then both arms go on (the sequence arm by the single call, then a sequence)
    to identical results.  The same for scans."""
    from loam_livox_b200.registration import Context
    capi = _capi()
    poses = S.trajectory(n_scans=6, n_static=2, speed=1.0)
    sizes = [N, N, N, 2 * N, N, N]
    frames = [[S.make_scan(n, p, seed=S.SEED + 3100 + k)] for k, (n, p) in enumerate(zip(sizes, poses))]
    stamps = [[100.0 + 0.1 * k] for k in range(6)]
    roomy = mapper(ctxs[0])
    feats = [[s.n_corner + s.n_surf for _, s in roomy.process_new_frame(f, t)] for f, t in zip(frames, stamps)]
    roomy.close()
    cap_f = max(max(feats[k]) for k in (0, 1, 2, 4, 5))
    assert max(feats[3]) > cap_f
    bad_piece = next(i for i, v in enumerate(feats[3]) if v > cap_f)
    small = [Context(0, max_scan_points=2 * N, max_features=cap_f) for _ in range(2)]
    try:
        ga, gb = mapper(small[0]), mapper(small[1])
        want = frames_single(ga, frames[:3], stamps[:3])
        status, n, want_partial = _raw_frame(ga, frames[3], stamps[3])
        assert status == capi.LL_ERR_CAPACITY and n == bad_piece
        status, done, n_pieces, got = _frames_call(gb, frames, stamps)
        assert status == capi.LL_ERR_CAPACITY and done == 3 and n_pieces[3] == bad_piece and n_pieces[4:] == [0, 0]
        assert got[:3] == want and got[3] == want_partial and state(ga) == state(gb)
        assert frames_single(ga, frames[4:], stamps[4:]) == frames_single(gb, frames[4:5], stamps[4:5]) + frames_seq(gb, frames[5:], stamps[5:])
        assert state(ga) == state(gb)
        ga.close(); gb.close()
    finally:
        for c in small:
            c.close()
    # scans: scan 3 over max_features; the sequence arm goes on by a sequence
    raws, ts = [f[0] for f in frames], [t[0] for t in stamps]
    roomy = mapper(ctxs[0])
    feats = [s.n_corner + s.n_surf for _, s in (roomy.process_new_scan(r, t) for r, t in zip(raws, ts))]
    roomy.close()
    cap_s = max(feats[k] for k in (0, 1, 2, 4, 5))
    assert feats[3] > cap_s
    small = [Context(0, max_scan_points=2 * N, max_features=cap_s) for _ in range(2)]
    try:
        ga, gb = mapper(small[0]), mapper(small[1])
        want = scans_single(ga, raws[:3], ts[:3])
        res, st = capi.RegResult(), capi.MapperStats()
        a = np.ascontiguousarray(raws[3])
        status_a = small[0]._lib.ll_mapper_process_scan(ga.h, C.c_void_p(a.ctypes.data), a.shape[0], capi.LL_FMT_XYZI16, capi.LL_HOST, ts[3], C.byref(res), C.byref(st))
        status, done, got = _scans_call(gb, raws, ts)
        assert status == status_a == capi.LL_ERR_CAPACITY and done == 3 and got == want and state(ga) == state(gb)
        assert scans_single(ga, raws[4:], ts[4:]) == scans_seq(gb, raws[4:], ts[4:]) and state(ga) == state(gb)
        ga.close(); gb.close()
    finally:
        for c in small:
            c.close()


def _raw_frame(gm, heads, stamps, odom_mode=1, cap=16, fmt=None, where=None, ns=None, null=None):
    """ll_mapper_process_frame directly: (status, *n_pieces, entries of the completed pieces)."""
    capi = _capi()
    arrs = [np.ascontiguousarray(h, np.float32) for h in heads]
    ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
    if null is not None:
        ptrs[null] = None
    sizes = (C.c_size_t * len(arrs))(*(ns or [a.shape[0] for a in arrs]))
    st = (C.c_double * len(arrs))(*stamps)
    res, stats, n = (capi.RegResult * 16)(), (capi.MapperStats * 16)(), C.c_int(-1)
    status = gm.ctx._lib.ll_mapper_process_frame(gm.h, len(arrs), ptrs, sizes, capi.LL_FMT_XYZI16 if fmt is None else fmt, capi.LL_HOST if where is None else where,
                                                 st, odom_mode, res, stats, cap, C.byref(n))
    return status, n.value, [entry(res[i], stats[i]) for i in range(n.value)]


@pytest.mark.gpu
def test_frame_graph_matches_eager_front_end(ctxs):
    """Frames of alternating sizes (N, N - 1).  One by one, every frame changes the shape of arena 0, so every front end runs eagerly.  In one
    sequence call frame f uses arena f & 1, whose shape repeats, so the front end is captured at frames 2 and 3 and replayed from then on.
    Results, launch counts and the end state are identical."""
    poses = S.trajectory(n_scans=8, n_static=2, speed=1.0)
    frames = [[S.make_scan(N, p, seed=S.SEED + 3300 + k)[: N - (k % 2)].copy()] for k, p in enumerate(poses)]
    stamps = [[100.0 + 0.1 * k] for k in range(8)]
    want, got = run_pair(ctxs, mapper, lambda g: frames_single(g, frames, stamps), lambda g: frames_seq(g, frames, stamps))
    assert got == want


def _continue(gm, frames, stamps, first_single):
    """(status, entries) per frame from here on: the first frame by the single call or not, the rest by sequence calls that restart after each
    input that fails."""
    out, i = [], 0
    if first_single:
        st, _, e = _raw_frame(gm, frames[0], stamps[0])
        out.append((st, e)); i = 1
    while i < len(frames):
        st, done, _, e = _frames_call(gm, frames[i:], stamps[i:])
        out += [(0, x) for x in e[:done]]
        if st != 0:
            out.append((st, e[done]))
        i += done + (st != 0)
    return out


@pytest.mark.gpu
def test_mapper_error_after_the_next_front_end_is_enqueued(ctxs):
    """Frame 4 is a scan scaled by 100 (same petals, nothing near the map): its registration fails (LL_ERR_NO_BLOCKS) inside the mapper step,
    after the front end of frame 5 has been enqueued.  The call returns the one-by-one arm's status, done count and entries, and the front end
    enqueued ahead is undone: going on from frame 5, by the single call or by a sequence, gives the one-by-one arm's results.  With deblur, so
    that the registrations read the extractor's time stamps.  The same for scans."""
    capi = _capi()
    frames, stamps = stream_frames(8, S.SEED + 3200)
    frames[4] = [frames[4][0] * np.array([100, 100, 100, 1], np.float32)]
    make = lambda c: mapper(c, init=2, if_motion_deblur=1)  # noqa: E731
    for first_single in (True, False):
        ga, gb = make(ctxs[0]), make(ctxs[1])
        want = [_raw_frame(ga, f, t) for f, t in zip(frames[:5], stamps[:5])]
        assert [st for st, _, _ in want] == [0, 0, 0, 0, capi.LL_ERR_NO_BLOCKS]
        status, done, n_pieces, got = _frames_call(gb, frames, stamps)
        assert status == capi.LL_ERR_NO_BLOCKS and done == 4 and n_pieces[4:] == [0, 0, 0, 0]
        assert got == [e for _, _, e in want] and state(ga) == state(gb)
        rest = [(st, e) for st, _, e in (_raw_frame(ga, f, t) for f, t in zip(frames[5:], stamps[5:]))]
        assert all(st == 0 and len(e) == 1 for st, e in rest)
        assert _continue(gb, frames[5:], stamps[5:], first_single) == rest and state(ga) == state(gb)
        ga.close(); gb.close()
    raws, ts = [f[0] for f in frames], [t[0] for t in stamps]
    ga, gb = make(ctxs[0]), make(ctxs[1])
    want = [_single_raw_scan_status(ga, r, t) for r, t in zip(raws[:5], ts[:5])]
    assert [st for st, _ in want] == [0, 0, 0, 0, capi.LL_ERR_NO_BLOCKS]
    status, done, got = _scans_call(gb, raws, ts)
    assert status == capi.LL_ERR_NO_BLOCKS and done == 4 and got == [e for _, e in want[:4]] and state(ga) == state(gb)
    assert scans_single(ga, raws[5:], ts[5:]) == scans_seq(gb, raws[5:], ts[5:]) and state(ga) == state(gb)
    ga.close(); gb.close()


def _single_raw_scan_status(gm, raw, stamp, fmt=None, where=None, n=None, null=False):
    capi = _capi()
    a = np.ascontiguousarray(raw, np.float32)
    res, st = capi.RegResult(), capi.MapperStats()
    status = gm.ctx._lib.ll_mapper_process_scan(gm.h, None if null else C.c_void_p(a.ctypes.data), a.shape[0] if n is None else n,
                                                capi.LL_FMT_XYZI16 if fmt is None else fmt, capi.LL_HOST if where is None else where, stamp, C.byref(res), C.byref(st))
    return status, entry(res, st)


@pytest.mark.gpu
def test_python_sequence_error_keeps_what_completed(ctxs):
    """Laser_mapping.process_new_frames raises SequenceError with the done count and the entries that completed."""
    from loam_livox_b200.registration import SequenceError
    frames, stamps = stream_frames(3, S.SEED + 3400)
    big = np.zeros((ctxs[1].cfg.max_scan_points, 4), np.float32)
    gb = mapper(ctxs[1])
    gb.process_new_frames(frames[:1], stamps[:1])
    with pytest.raises(SequenceError) as e:   # a validation error: nothing done
        gb.process_new_frames([frames[1], [np.concatenate([big, big[:1]])]], stamps[1:3])
    assert e.value.done == 0 and e.value.results == [[]] and e.value.status == _capi().LL_ERR_CAPACITY
    gb.close()
