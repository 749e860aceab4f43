"""Every entry point of the device front end against the oracle, bit for bit: the features a call registers (ll_features_to_pointcloud2, both
classes), their counts, the call's status and whether the input was dropped.  The edges are where the entry points' rules differ:
ll_scan_to_pose never drops a whole scan and drops a piece of a scan with <= 5 petals; ll_frame_to_pose takes a head iff it has >= 5 points
(and, for a piece, > 5 petals); the streaming mapper takes a head iff it has points and > 5 petals."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from loam_livox_b200 import synthetic as S  # noqa: E402
import piecewise_oracle as PO  # noqa: E402

N = 24000
LEAF = (0.1, 0.2, 0.1, 0.4)   # extractor corner / surface, mapping corner / surface


def _capi():
    from loam_livox_b200 import capi
    return capi


def pipe(whole=1, pieces=3, use_piece=0):
    return _capi().PipelineCfg(pieces=pieces, use_piece=use_piece, extractor_leaf_corner=LEAF[0], extractor_leaf_surf=LEAF[1],
                               mapping_leaf_corner=LEAF[2], mapping_leaf_surf=LEAF[3], whole_frame=whole)


@pytest.fixture(scope="module")
def match_map(ctx):
    from loam_livox_b200.registration import Map
    m = Map(ctx, *S.make_map(5000, 45000))
    yield m
    m.release()


@pytest.fixture
def fresh(ctx, oracle):
    """The device extractor reset and a fresh oracle extractor: both keep the same time-stamp bookkeeping from here on."""
    ctx._lib.ll_extract_reset(ctx.h)
    return oracle.Extractor()


def voxel_chains(oracle, c, s):
    return oracle.voxel_grid(oracle.voxel_grid(c, LEAF[0]), LEAF[2]), oracle.voxel_grid(oracle.voxel_grid(s, LEAF[1]), LEAF[3])


def head_features(ex, raw, stamp, pc):
    """(corner, surface, petals) of one head before the VoxelGrids: bounds 0 ... 1, or piece use_piece of the piece bounds."""
    petals = ex.extract(raw, stamp)
    if pc.whole_frame:
        c, s, _ = ex.get_features(0.0, 1.0)
    else:
        start, end = ex.piece_bounds(pc.pieces)
        c, s, _ = ex.get_features(start[pc.use_piece], end[pc.use_piece])
    return c, s, petals


def want_scan(oracle, ex, raw, stamp, pc):
    """ll_scan_to_pose on the oracle: (corner, surface, dropped)."""
    c, s, petals = head_features(ex, raw, stamp, pc)
    return (*voxel_chains(oracle, c, s), bool(not pc.whole_frame and petals <= 5))


def want_frame(oracle, ex, heads, stamps, pc):
    """ll_frame_to_pose on the oracle: one extractor over the heads in turn, the clouds of the heads that count summed, then the VoxelGrids."""
    cs, ss = [], []
    for raw, stamp in zip(heads, stamps):
        c, s, petals = head_features(ex, raw, stamp, pc)
        if raw.shape[0] >= 5 and (pc.whole_frame or petals > 5):
            cs.append(c); ss.append(s)
    z = np.zeros((0, 4), np.float32)
    return voxel_chains(oracle, np.concatenate(cs) if cs else z, np.concatenate(ss) if ss else z)


def features(ctx):
    from loam_livox_b200.registration import features_to_pointcloud2
    return tuple(np.frombuffer(features_to_pointcloud2(ctx, k), np.float32).reshape(-1, 4) for k in (0, 1))


def reg_state():
    return _capi().default_reg_state()


def scan_call(ctx, m, raw, stamp, pc, fmt=None, where=None, n=None):
    """ll_scan_to_pose: (status, registered, n_corner, n_surf)."""
    capi = _capi()
    if where is None:
        raw = np.ascontiguousarray(raw, np.float32)
        ptr, n, where, fmt = raw.ctypes.data, raw.shape[0], capi.LL_HOST, capi.LL_FMT_XYZI16 if raw.shape[1] == 4 else capi.LL_FMT_PCL32
    else:
        ptr = raw
    res, nc, ns = capi.RegResult(), C.c_int(), C.c_int()
    st = ctx._lib.ll_scan_to_pose(ctx.h, m.h, ptr, n, fmt, where, C.c_double(stamp), C.byref(pc), C.byref(reg_state()), C.byref(res), C.byref(nc), C.byref(ns))
    return st, res.registered, nc.value, ns.value


def frame_call(ctx, m, heads, stamps, pc, where=None, ns=None, fmt=None):
    """ll_frame_to_pose: (status, registered, n_corner, n_surf)."""
    capi = _capi()
    k = len(heads)
    if where is None:
        arrs = [np.ascontiguousarray(h, np.float32) for h in heads]
        ptrs, ns, where = [a.ctypes.data for a in arrs], [a.shape[0] for a in arrs], capi.LL_HOST
        fmt = capi.LL_FMT_XYZI16 if arrs[0].shape[1] == 4 else capi.LL_FMT_PCL32
    else:
        ptrs = heads
    res, nc, nsf = capi.RegResult(), C.c_int(), C.c_int()
    st = ctx._lib.ll_frame_to_pose(ctx.h, m.h, k, (C.c_void_p * k)(*ptrs), (C.c_size_t * k)(*ns), fmt, where, (C.c_double * k)(*stamps), C.byref(pc),
                                   C.byref(reg_state()), C.byref(res), C.byref(nc), C.byref(nsf))
    return st, res.registered, nc.value, nsf.value


def check_scan(ctx, oracle, m, ex, raw, stamp, pc, **kw):
    """One ll_scan_to_pose against the oracle; returns the registered features."""
    capi = _capi()
    c, s, dropped = want_scan(oracle, ex, raw, stamp, pc)
    st, registered, nc, ns = scan_call(ctx, m, raw, stamp, pc, **kw)
    assert (nc, ns) == (c.shape[0], s.shape[0])
    if dropped:
        assert st == capi.LL_OK and registered == 0
        return None
    assert st == capi.LL_ERR_NO_BLOCKS if nc + ns == 0 else st in (capi.LL_OK, capi.LL_ERR_NO_BLOCKS)
    got = features(ctx)
    assert got[0].tobytes() == c.tobytes() and got[1].tobytes() == s.tobytes()
    return got


def check_frame(ctx, oracle, m, ex, heads, stamps, pc, **kw):
    capi = _capi()
    c, s = want_frame(oracle, ex, heads, stamps, pc)
    st, registered, nc, ns = frame_call(ctx, m, heads, stamps, pc, **kw)
    assert (nc, ns) == (c.shape[0], s.shape[0])
    assert st == capi.LL_ERR_NO_BLOCKS if nc + ns == 0 else st in (capi.LL_OK, capi.LL_ERR_NO_BLOCKS)
    got = features(ctx)
    assert got[0].tobytes() == c.tobytes() and got[1].tobytes() == s.tobytes()
    return got


def scan(k, n=N):
    return S.make_scan(n, S.default_pose(), seed=S.SEED + 3000 + k)


def few_petals(oracle, raw, petals):
    ex = oracle.Extractor()
    for m in range(50, raw.shape[0], 20):
        if ex.extract(raw[:m], 100.0) == petals:
            return raw[:m].copy()
    raise AssertionError(petals)


SELECTIONS = [dict(whole=1), dict(whole=0, use_piece=0), dict(whole=0, use_piece=1), dict(whole=0, use_piece=2)]


@pytest.mark.gpu
@pytest.mark.parametrize("sel", SELECTIONS, ids=["whole", "piece0of3", "piece1of3", "piece2of3"])
def test_scan_and_one_head_frame(ctx, oracle, match_map, fresh, sel):
    """ll_scan_to_pose, then ll_frame_to_pose with one head on the next scan, each against the oracle."""
    pc = pipe(**sel)
    check_scan(ctx, oracle, match_map, fresh, scan(0), 100.0, pc)
    check_frame(ctx, oracle, match_map, fresh, [scan(0)], [100.1], pc)


@pytest.mark.gpu
@pytest.mark.parametrize("petals", [5, 6])
@pytest.mark.parametrize("whole", [0, 1])
def test_scan_petal_edge(ctx, oracle, match_map, fresh, petals, whole):
    """A scan of 5 petals is dropped under whole_frame 0 and registered under 1; 6 petals are registered under both."""
    raw = few_petals(oracle, scan(1), petals)
    got = check_scan(ctx, oracle, match_map, fresh, raw, 100.0, pipe(whole=whole))
    assert (got is None) == (petals == 5 and whole == 0)


@pytest.mark.gpu
def test_sixteen_overlapping_pieces(ctx, oracle, match_map, fresh):
    """16 pieces of scans with 6 ... 8 petals (bounds clamp, pieces overlap): several use_piece through both calls."""
    for k, use in enumerate((0, 5, 9, 15)):
        raw = few_petals(oracle, scan(10 + k), 6 + k % 3)
        check_scan(ctx, oracle, match_map, fresh, raw, 100.0 + 0.2 * k, pipe(whole=0, pieces=16, use_piece=use))
        check_frame(ctx, oracle, match_map, fresh, [raw], [100.1 + 0.2 * k], pipe(whole=0, pieces=16, use_piece=use))


@pytest.mark.gpu
@pytest.mark.parametrize("whole", [0, 1])
def test_tiny_heads(ctx, oracle, match_map, fresh, whole):
    """Heads of 0, 1, 4, 5 and 6 points: alone through ll_scan_to_pose, and between two scans through ll_frame_to_pose (>= 5 points count)."""
    t = 100.0
    for n in (0, 1, 4, 5, 6):
        tiny = scan(20 + n)[:n]
        check_scan(ctx, oracle, match_map, fresh, tiny, t, pipe(whole=whole)); t += 0.1
        check_frame(ctx, oracle, match_map, fresh, [scan(30, 12000), tiny, scan(31, 12000)], [t, t + 0.01, t + 0.02], pipe(whole=whole)); t += 0.1


@pytest.mark.gpu
@pytest.mark.parametrize("sel", SELECTIONS[:2], ids=["whole", "piece0of3"])
def test_eight_heads_one_dropped(ctx, oracle, match_map, fresh, sel):
    """8 heads, one of 50 points and no petals: it counts in a whole frame (>= 5 points) and not in a piece (<= 5 petals)."""
    heads = [scan(40 + h, 6000) for h in range(8)]
    heads[5] = few_petals(oracle, scan(48), 0)
    check_frame(ctx, oracle, match_map, fresh, heads, [100.0 + 0.01 * h for h in range(8)], pipe(**sel))


def check_against(ctx, want, call):
    """A call's (status, registered, n_corner, n_surf) and registered features against the oracle's (corner, surface, ...)."""
    capi = _capi()
    st, _, nc, ns = call
    assert st in (capi.LL_OK, capi.LL_ERR_NO_BLOCKS) and (nc, ns) == (want[0].shape[0], want[1].shape[0])
    got = features(ctx)
    assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes()


@pytest.mark.gpu
def test_formats_and_device_inputs(ctx, oracle, match_map, fresh):
    """PCL32, STRIDED and device inputs of both calls against the oracle."""
    import torch
    capi = _capi()
    raws = [scan(50 + k, 12000) for k in range(3)]
    pcl = [np.concatenate([r[:, :3], np.zeros((r.shape[0], 1), np.float32), r[:, 3:4], np.zeros((r.shape[0], 3), np.float32)], axis=1) for r in raws]
    dev = [torch.from_numpy(r).cuda() for r in raws]
    torch.cuda.synchronize()
    t = 100.0
    for sel in SELECTIONS[:2]:
        pc = pipe(**sel)
        check_against(ctx, want_scan(oracle, fresh, raws[0], t, pc), scan_call(ctx, match_map, pcl[0], t, pc)); t += 0.1
        stamps = [t, t + 0.01, t + 0.02]; t += 0.1
        check_against(ctx, want_frame(oracle, fresh, raws, stamps, pc), frame_call(ctx, match_map, pcl, stamps, pc))
        check_against(ctx, want_scan(oracle, fresh, raws[0], t, pc),
                      scan_call(ctx, match_map, dev[0].data_ptr(), t, pc, fmt=capi.LL_FMT_XYZI16, where=capi.LL_DEVICE, n=raws[0].shape[0])); t += 0.1
        stamps = [t, t + 0.01, t + 0.02]; t += 0.1
        check_against(ctx, want_frame(oracle, fresh, raws, stamps, pc),
                      frame_call(ctx, match_map, [d.data_ptr() for d in dev], stamps, pc, where=capi.LL_DEVICE, ns=[r.shape[0] for r in raws], fmt=capi.LL_FMT_XYZI16))
    rec = np.zeros((raws[0].shape[0], 5), np.float32)
    rec[:, 0:3], rec[:, 4] = raws[0][:, :3], raws[0][:, 3]

    def strided(call):   # the call on the records, the features read back in the default layout
        ctx.set_point_layout(20, 0, 4, 8, 16, capi.LL_I_FLOAT32)
        try:
            return call()
        finally:
            ctx.set_point_layout(16)
    check_against(ctx, want_scan(oracle, fresh, raws[0], t, pipe()),
                  strided(lambda: scan_call(ctx, match_map, rec.ctypes.data, t, pipe(), fmt=capi.LL_FMT_STRIDED, where=capi.LL_HOST, n=rec.shape[0])))
    stamps = [t + 0.1, t + 0.11]
    check_against(ctx, want_frame(oracle, fresh, [raws[0], raws[0]], stamps, pipe()),
                  strided(lambda: frame_call(ctx, match_map, [rec.ctypes.data] * 2, stamps, pipe(), where=capi.LL_HOST, ns=[rec.shape[0]] * 2,
                                             fmt=capi.LL_FMT_STRIDED)))


@pytest.mark.gpu
def test_repeated_shape_then_changed(ctx, oracle, match_map, fresh):
    """The same shape three times (eager, captured, replayed), then a changed one, through both calls."""
    t = 100.0
    for k in range(4):
        n = N if k < 3 else N - 1000
        for sel in SELECTIONS[:2]:
            check_scan(ctx, oracle, match_map, fresh, scan(60 + k, n), t, pipe(**sel)); t += 0.1
            check_frame(ctx, oracle, match_map, fresh, [scan(70 + k, n // 2), scan(80 + k, n // 3)], [t, t + 0.01], pipe(**sel)); t += 0.1


@pytest.mark.gpu
def test_mapper_front_ends(ctx, oracle):
    """The streaming mapper's scans (whole_frame 1 and 0, one of 5 petals) and frames (3 heads, one without petals; the same shape three times,
    then a changed one): the feature counts of every input against the oracle, and the features of every registered scan and of the last
    registered piece of every frame (the features a mapper registers are the context's last ones)."""
    from loam_livox_b200.registration import Laser_mapping
    capi = _capi()
    registered = 0
    for whole in (1, 0):
        gm = Laser_mapping(ctx, reg=capi.default_reg_state(mapping_init_accumulate_frames=2), pipeline=pipe(whole=whole))
        ex = oracle.Extractor()
        raws = [scan(90), few_petals(oracle, scan(91), 5), scan(92), scan(93), scan(94, N - 500)]
        for k, raw in enumerate(raws):
            c, s, _ = want_scan(oracle, ex, raw, 100.0 + 0.1 * k, pipe(whole=whole))
            res, st = gm.process_new_scan(raw, 100.0 + 0.1 * k)
            assert (st.n_corner, st.n_surf) == (c.shape[0], s.shape[0]), (whole, k)
            if res.registered:
                registered += 1
                got = features(ctx)
                assert got[0].tobytes() == c.tobytes() and got[1].tobytes() == s.tobytes(), (whole, k)
        gm.close()
    gm = Laser_mapping(ctx, reg=capi.default_reg_state(mapping_init_accumulate_frames=2), pipeline=pipe(whole=0))
    ex = oracle.Extractor()
    for k in range(4):
        heads = [scan(100 + 3 * k + h, 8000 if k < 3 else 7000) for h in range(3)]
        heads[1] = few_petals(oracle, heads[1], 0) if k == 3 else heads[1]
        stamps = [100.0 + 0.1 * k] * 3
        parts, live = PO.frame_pieces(ex, heads, stamps, 3)
        got = gm.process_new_frame(heads, stamps)
        assert len(got) == (3 if live else 0)
        last = None
        for (res, st), (c, s, _) in zip(got, parts):
            c, s = voxel_chains(oracle, c, s)
            assert (st.n_corner, st.n_surf) == (c.shape[0], s.shape[0]), k
            last = (c, s) if res.registered else last
        if last is not None:
            registered += 1
            f = features(ctx)
            assert f[0].tobytes() == last[0].tobytes() and f[1].tobytes() == last[1].tobytes(), k
    gm.close()
    assert registered >= 4
