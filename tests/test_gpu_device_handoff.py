"""ll_scan_to_pose starts the ICP loop from the front end's device-side counts (no host read in between): its result must equal, bit for bit,
ll_register on the same features (the host-sized path), in every RegResult field but the gpu_ms_* timings, with the same status and error.
The features are read back with ll_features_to_pointcloud2 after the call, and registered again on the same context from the same state."""
import ctypes as C
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from loam_livox_b200 import synthetic as S  # noqa: E402

pytestmark = pytest.mark.gpu

N = 24000
TIMINGS = {"gpu_ms_total", "gpu_ms_knn", "gpu_ms_sort", "gpu_ms_knn_all", "gpu_ms_solve_all", "gpu_ms_select_all"}


def _capi():
    from loam_livox_b200 import capi
    return capi


def pipe(whole=1, pieces=3, use_piece=0):
    return _capi().PipelineCfg(pieces=pieces, use_piece=use_piece, extractor_leaf_corner=0.1, extractor_leaf_surf=0.2, mapping_leaf_corner=0.1,
                               mapping_leaf_surf=0.4, whole_frame=whole)


@pytest.fixture(scope="module")
def maps():
    return S.make_map(5000, 45000)


def fields(r):
    out = {}
    for name, _ in r._fields_:
        if name in TIMINGS:
            continue
        v = getattr(r, name)
        out[name] = tuple(v) if hasattr(v, "__len__") else v
    return out


def state(guess, **kw):
    return _capi().default_reg_state(q_w_last=guess.q, t_w_last=guess.t, q_w_curr=guess.q, t_w_curr=guess.t, **kw)


def call(ctx, m, raw, stamp, pc, st):
    """ll_scan_to_pose: (status, error, result fields, nc, ns, features)."""
    from loam_livox_b200.registration import features_to_pointcloud2
    capi = _capi()
    pts = np.ascontiguousarray(raw, np.float32)
    res = capi.RegResult()
    nc, ns = C.c_int(), C.c_int()
    code = ctx._lib.ll_scan_to_pose(ctx.h, m.h, pts.ctypes.data, pts.shape[0], capi.LL_FMT_XYZI16, capi.LL_HOST, float(stamp), C.byref(pc), C.byref(st),
                                    C.byref(res), C.byref(nc), C.byref(ns))
    err = ctx._lib.ll_last_error(ctx.h).decode()
    feats = tuple(np.frombuffer(features_to_pointcloud2(ctx, k), np.float32).reshape(-1, 4).copy() for k in (0, 1))
    return code, err, fields(res), nc.value, ns.value, feats


def register(ctx, m, corner, surf, st):
    capi = _capi()
    c = np.ascontiguousarray(corner, np.float32)
    s = np.ascontiguousarray(surf, np.float32)
    res = capi.RegResult()
    code = ctx._lib.ll_register(ctx.h, m.h, c.ctypes.data, c.shape[0], s.ctypes.data, s.shape[0], capi.LL_FMT_XYZI16, capi.LL_HOST, C.byref(st), C.byref(res))
    return code, ctx._lib.ll_last_error(ctx.h).decode(), fields(res)


def check_equals_register(ctx, m, raw, stamp, pc, st):
    code, err, got, nc, ns, (fc, fs) = call(ctx, m, raw, stamp, pc, st)
    assert (fc.shape[0], fs.shape[0]) == (nc, ns)
    rcode, rerr, want = register(ctx, m, fc, fs, st)
    assert (code, got) == (rcode, want)
    if code != 0:
        assert err == rerr
    return code, got, nc, ns


def test_c2_like_scans_eager_and_graph_replayed(maps):
    """The first call of a shape runs the front end eagerly, the second captures it, the third replays it."""
    from loam_livox_b200.registration import Context, Map
    ctx = Context(0, max_scan_points=N, max_features=N)
    m = Map(ctx, *maps)
    pose = S.default_pose()
    raw = S.make_scan(N, pose)
    for k in range(4):
        g = S.perturb_pose(pose, np.random.default_rng(10 + k), dt=0.05, dang_deg=1.0)
        code, got, nc, ns = check_equals_register(ctx, m, raw, 100.0 + 0.1 * k, pipe(), state(g))
        assert code == 0 and got["registered"] == 1 and nc + ns > 1000
    m.release(); ctx.close()


@pytest.mark.parametrize("n", [40, 200, 1500, 6000, 15000])
def test_scan_sizes(maps, n):
    """Scans of different sizes give feature counts across the solver's tile / CTA splits (one CTA, part-filled tiles, whole ones)."""
    from loam_livox_b200.registration import Context, Map
    ctx = Context(0, max_scan_points=N, max_features=N)
    m = Map(ctx, *maps)
    pose = S.default_pose()
    g = S.perturb_pose(pose, np.random.default_rng(3), dt=0.03, dang_deg=0.5)
    check_equals_register(ctx, m, S.make_scan(n, pose, seed=7 + n), 100.0, pipe(), state(g))
    m.release(); ctx.close()


@pytest.mark.parametrize("cap", [150, 700])
def test_residual_cap_binds(maps, cap):
    """More features than 2 x maximum_allow_residual_block: the pre-skip and the drop rule run from the device counts."""
    from loam_livox_b200.registration import Context, Map
    ctx = Context(0, max_scan_points=N, max_features=N)
    m = Map(ctx, *maps)
    pose = S.default_pose()
    g = S.perturb_pose(pose, np.random.default_rng(5), dt=0.03, dang_deg=0.5)
    code, got, nc, ns = check_equals_register(ctx, m, S.make_scan(N, pose), 100.0, pipe(), state(g, maximum_allow_residual_block=cap, rng_seed=11))
    assert nc + ns > 2 * cap
    m.release(); ctx.close()


def test_deblur(maps):
    from loam_livox_b200.registration import Context, Map
    ctx = Context(0, max_scan_points=N, max_features=N)
    m = Map(ctx, *maps)
    pose = S.default_pose()
    g = S.perturb_pose(pose, np.random.default_rng(6), dt=0.03, dang_deg=0.5)
    check_equals_register(ctx, m, S.make_scan(N, pose), 100.0, pipe(), state(g, if_motion_deblur=1))
    m.release(); ctx.close()


def test_all_nan_scan_reports_no_features(maps):
    from loam_livox_b200.registration import Context, Map
    capi = _capi()
    ctx = Context(0, max_scan_points=N, max_features=N)
    small = Context(0, max_scan_points=N, max_features=N - 1)   # max_features < max_scan_points: the host-sized path
    raw = np.full((5000, 4), np.nan, np.float32)
    g = S.default_pose()
    outs = []
    for c in (ctx, small):
        m = Map(c, *maps)
        code, err, got, nc, ns, _ = call(c, m, raw, 100.0, pipe(), state(g))
        outs.append((code, err, got, nc, ns))
        m.release()
    assert outs[0] == outs[1]
    assert outs[0][0] == capi.LL_ERR_NO_BLOCKS and outs[0][1] == "no features"
    ctx.close(); small.close()


def test_dropped_piece_and_fallback_context_agree(maps):
    """whole_frame = 0 on a scan with <= 5 petals is dropped: same status, error, counts and result as the host-sized path, and the features of
    the previous call stay.  Then a normal scan on both contexts: the same result."""
    from loam_livox_b200.registration import Context, Map
    dev = Context(0, max_scan_points=N, max_features=N)
    host = Context(0, max_scan_points=N, max_features=N - 1)
    pose = S.default_pose()
    g = S.perturb_pose(pose, np.random.default_rng(8), dt=0.03, dang_deg=0.5)
    big = S.make_scan(N, pose)
    tiny = S.make_scan(30, pose, seed=99)
    outs = []
    for c in (dev, host):
        m = Map(c, *maps)
        c._lib.ll_extract_reset(c.h)
        a = call(c, m, big, 100.0, pipe(), state(g))
        b = call(c, m, tiny, 100.1, pipe(whole=0), state(g))
        outs.append((a, b))
        m.release()
    (a0, b0), (a1, b1) = outs
    assert a0[:5] == a1[:5] and all(np.array_equal(x, y) for x, y in zip(a0[5], a1[5]))
    assert b0[:5] == b1[:5] and b0[1] == "frame dropped: <= 5 petals"
    assert all(np.array_equal(x, y) for x, y in zip(b0[5], a0[5]))   # a dropped scan leaves the previous features
    dev.close(); host.close()


def test_two_contexts_on_two_host_threads_share_one_map(maps):
    from loam_livox_b200.registration import Context, Map
    ctxs = [Context(0, max_scan_points=N, max_features=N) for _ in range(2)]
    m = Map(ctxs[0], *maps)
    pose = S.default_pose()
    raw = S.make_scan(N, pose)
    guesses = [S.perturb_pose(pose, np.random.default_rng(100 + k), dt=0.05, dang_deg=1.0) for k in range(4)]

    def run(c, k):
        c._lib.ll_extract_reset(c.h)
        code, err, got, nc, ns, _ = call(c, m, raw, 100.0, pipe(), state(guesses[k]))
        return code, got, nc, ns
    alone = [run(ctxs[0], k) for k in range(len(guesses))]
    out = [[None] * len(guesses) for _ in range(2)]
    errs = []

    def worker(w):
        try:
            for _ in range(3):
                for k in (range(len(guesses)) if w == 0 else reversed(range(len(guesses)))):
                    out[w][k] = run(ctxs[w], k)
        except Exception as e:   # noqa: BLE001
            errs.append(e)
    ths = [threading.Thread(target=worker, args=(w,)) for w in range(2)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    assert not errs, errs
    assert out[0] == alone and out[1] == alone
    m.release()
    for c in ctxs:
        c.close()
