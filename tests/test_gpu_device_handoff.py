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


# ---------------------------------------------------------------------------------------------- exact feature counts (ll_register_dev_counts)
# ll_register_dev_counts puts caller-given features where the front end leaves them and runs ll_scan_to_pose's registration on the device
# counts: the capacity-sized spatial sort (padding keys past M), the kNN instance that reads the counts, and the solver launched on T CTAs with
# the capacity's shared memory, which recomputes the split, cap_check and the K10 hash-set mask from the device M.  Every count below is
# derived from T = min(SMs, LL_SYNC_ROWS) and the solver's split, restated here.
SYNC_ROWS = 160       # LL_SYNC_ROWS: the solver's grid has at most this many CTAs
SOLVE_THREADS = 256   # slots per solver tile at most


def solve_grid(ncta, M):
    """solve.cu's solve_grid: (tile, tiles_per_cta, grid) for M slots over ncta CTAs."""
    M1 = max(M, 1)
    tile = min(((M1 + ncta - 1) // ncta + 31) // 32 * 32, SOLVE_THREADS)
    tiles = (M1 + tile - 1) // tile
    grid = min(tiles, ncta)
    return tile, (tiles + grid - 1) // grid, grid


def n_ctas():
    import torch
    return min(torch.cuda.get_device_properties(0).multi_processor_count, SYNC_ROWS)


# the counts across the device split, as functions of T and the capacity C
EDGES = {"1": lambda T, C: 1, "2": lambda T, C: 2, "31": lambda T, C: 31, "32": lambda T, C: 32, "33": lambda T, C: 33,
         "32(T-1)": lambda T, C: 32 * (T - 1), "32T": lambda T, C: 32 * T, "32T+1": lambda T, C: 32 * T + 1,
         "256T-1": lambda T, C: 256 * T - 1, "256T": lambda T, C: 256 * T, "256T+1": lambda T, C: 256 * T + 1,
         "512T": lambda T, C: 512 * T, "512T+1": lambda T, C: 512 * T + 1, "C-1": lambda T, C: C - 1, "C": lambda T, C: C}


def splits(M):
    """(corners, surfaces): one class empty, one feature in a class, and a realistic 1:9."""
    return sorted({(0, M), (M, 0), (1, M - 1), (M - 1, 1), (M // 10, M - M // 10)})


class Big:
    """One context of capacity C >= 3 * 256 T + 1000 (the solver launch always has T CTAs and shared memory for >= 3 tiles each), its map,
    and feature pools of C corners and C surfaces sampled from the same scene."""

    def __init__(self):
        from loam_livox_b200.registration import Context, Map
        self.T = n_ctas()
        self.C = max(110000, 3 * 256 * self.T + 1000)
        self.mc, self.ms = S.make_map(20000, 180000)
        self.pose = S.default_pose()
        self.fc, self.fs = S.make_features(self.C, self.C, self.pose)
        self.guess = S.perturb_pose(self.pose, np.random.default_rng(3), dt=0.03, dang_deg=0.5)
        self.ctx = Context(0, max_scan_points=self.C, max_features=self.C)
        self.m = Map(self.ctx, self.mc, self.ms)

    def context(self, cap):
        from loam_livox_b200.registration import Context, Map
        c = Context(0, max_scan_points=cap, max_features=cap)
        return c, Map(c, self.mc, self.ms)

    def feats(self, nc, ns):
        return self.fc[:nc], self.fs[:ns]


@pytest.fixture(scope="module")
def big():
    b = Big()
    yield b
    b.m.release(); b.ctx.close()


def dev_counts(ctx, m, corner, surf, st):
    """ll_register_dev_counts: (status, error, result fields)."""
    capi = _capi()
    c = np.ascontiguousarray(corner, np.float32)
    s = np.ascontiguousarray(surf, np.float32)
    res = capi.RegResult()
    code = ctx._lib.ll_register_dev_counts(ctx.h, m.h, c.ctypes.data, c.shape[0], s.ctypes.data, s.shape[0], capi.LL_FMT_XYZI16, capi.LL_HOST,
                                           C.byref(st), C.byref(res))
    return code, ctx._lib.ll_last_error(ctx.h).decode(), fields(res)


def last_features(ctx):
    from loam_livox_b200.registration import features_to_pointcloud2
    return tuple(np.frombuffer(features_to_pointcloud2(ctx, k), np.float32).reshape(-1, 4) for k in (0, 1))


def check_dev_equals_register(ctx, m, corner, surf, st):
    """The device-count path and ll_register on the same context, features and state: the same status, error text and result bits."""
    code, err, got = dev_counts(ctx, m, corner, surf, st)
    if code == 0:   # the registration's features are the caller's, in their order
        fc, fs = last_features(ctx)
        assert np.array_equal(fc, corner, equal_nan=True) and np.array_equal(fs, surf, equal_nan=True)
    rcode, rerr, want = register(ctx, m, corner, surf, st)
    assert (code, got) == (rcode, want)
    if code != 0:
        assert err == rerr
    return code, err, got


def check_oracle(oracle, b, corner, surf, got, **kw):
    """test_register_pose_parity's bars against the CPU oracle."""
    g = b.guess
    p = oracle.default_params(q_w_last=g.q, t_w_last=g.t, q_w_curr=g.q, t_w_curr=g.t, **kw)
    ost, ores = oracle.register(b.mc, b.tc, b.ms, b.ts, corner, surf, p)
    assert got["status"] == ost and got["registered"] == 1 and got["icp_iterations"] == ores.icp_iterations
    assert (got["corner_used"], got["surf_used"], got["num_residual_blocks"]) == (ores.corner_used, ores.surf_used, ores.num_residual_blocks)
    dt = np.linalg.norm(np.array(got["t_w_curr"]) - np.array(ores.t_w_curr))
    da = S.quat_angle(np.array(got["q_w_curr"]), np.array(ores.q_w_curr))
    assert dt < 1e-7 and da < 1e-7, (dt, da)
    assert abs(got["final_cost"] - ores.final_cost) <= 1e-7 * ores.final_cost
    assert abs(got["inlier_threshold"] - ores.inlier_threshold) <= 1e-7 * ores.inlier_threshold


@pytest.fixture(scope="module")
def trees(big, oracle):
    big.tc, big.ts = oracle.KdTree(big.mc), oracle.KdTree(big.ms)
    return big


def test_the_counts_sit_on_the_split_edges(big):
    """The counts below are where the solver's split changes: grids short of T, the tile growing by 32, the second and third tile per CTA."""
    T, C = big.T, big.C
    E = {k: f(T, C) for k, f in EDGES.items()}
    assert solve_grid(T, C)[2] == T and solve_grid(T, C)[1] >= 3
    assert solve_grid(T, E["33"]) == (32, 1, 2) and solve_grid(T, E["32(T-1)"]) == (32, 1, T - 1)
    assert solve_grid(T, E["32T"]) == (32, 1, T) and solve_grid(T, E["32T+1"])[0] == 64
    assert solve_grid(T, E["256T"]) == (256, 1, T) and solve_grid(T, E["256T+1"]) == (256, 2, T)
    assert solve_grid(T, E["512T"]) == (256, 2, T) and solve_grid(T, E["512T+1"]) == (256, 3, T)


@pytest.mark.parametrize("edge", list(EDGES))
def test_exact_counts_across_the_device_split(big, edge):
    """Every split of M = edge into corners and surfaces: the device-count path equals ll_register, bit for bit."""
    M = EDGES[edge](big.T, big.C)
    st = state(big.guess)
    for nc, ns in splits(M):
        check_dev_equals_register(big.ctx, big.m, *big.feats(nc, ns), st)


def test_capacity_equal_to_one_tile_per_cta_and_one_slot(big):
    """Capacity 256 T + 1: the launch's split (2 tiles per CTA) is the device split at M = capacity."""
    T = big.T
    cap = 256 * T + 1
    ctx, m = big.context(cap)
    st = state(big.guess)
    for M in sorted({f(T, cap) for f in EDGES.values()} - {512 * T, 512 * T + 1}):
        for nc, ns in splits(M):
            check_dev_equals_register(ctx, m, *big.feats(nc, ns), st)
    m.release(); ctx.close()


@pytest.mark.parametrize("edge", ["32(T-1)", "32T+1", "256T+1"])
def test_split_edges_against_the_oracle(trees, oracle, edge):
    """Bit equality with ll_register cannot see a fault in the split both share: at a grid short of T, at the first 64-slot tile and at the
    second tile per CTA the result also matches the CPU oracle."""
    b = trees
    M = EDGES[edge](b.T, b.C)
    corner, surf = b.feats(M // 10, M - M // 10)
    code, _, got = check_dev_equals_register(b.ctx, b.m, corner, surf, state(b.guess))
    assert code == 0
    check_oracle(oracle, b, corner, surf, got)


def cap_seed(cap, lib):
    """A seed for which ICP iteration 0 draws at least one drop among cap + 1 blocks and at least one pre-skip among 2 cap + 1 corners and
    among 2 cap + 1 surfaces (the rules' float arithmetic): the +1 counts then change the result."""
    f32 = np.float32
    for seed in range(100):
        u = lambda stream, n: np.array([lib.ll_cap_uniform(seed, 0, stream, i) for i in range(n)], np.float32)
        drop = (u(2, cap + 1) > f32(cap) / f32(cap + 1)).any()
        skip = [(u(k, 2 * cap + 1) * f32(2 * cap + 1) > f32(2 * cap)).any() for k in (0, 1)]
        if drop and all(skip):
            return seed
    raise AssertionError("no seed in 0 ... 99")


def test_residual_cap_and_pre_skip_edges(trees, oracle):
    """maximum_allow_residual_block = cap: M = cap and cap + 1 all surfaces (every one a block: the drop rule behind cap_check fires at cap + 1
    only); corners = 2 cap and 2 cap + 1 beside fewer surfaces, then the reverse (the pre-skip, each class by its own device count)."""
    from loam_livox_b200.registration import Point_cloud_registration
    b = trees
    cap = 700
    seed = cap_seed(cap, b.ctx._lib)
    kw = dict(maximum_allow_residual_block=cap, rng_seed=seed)
    st = state(b.guess, **kw)
    reg = Point_cloud_registration(b.ctx, **kw)
    reg.set_pose(b.guess.q, b.guess.t)
    assert int((reg.build_blocks(b.m, *b.feats(0, cap + 1))[0] != 0).sum()) == cap + 1
    cases = [((0, cap), False), ((0, cap + 1), True),
             ((2 * cap, 2 * cap - 100), False), ((2 * cap + 1, 2 * cap - 100), True),
             ((2 * cap - 100, 2 * cap), False), ((2 * cap - 100, 2 * cap + 1), True)]
    for (nc, ns), with_oracle in cases:
        corner, surf = b.feats(nc, ns)
        code, _, got = check_dev_equals_register(b.ctx, b.m, corner, surf, st)
        if with_oracle:
            assert code == 0
            check_oracle(oracle, b, corner, surf, got, **kw)


@pytest.mark.parametrize("M", [512, 513, 1024, 1025])
def test_k10_hash_set_size_from_the_device_count(big, M):
    """The table is laid out for the capacity; the device M sets the mask (1024 slots up to M = 512, then 2048, 4096).  A third of the surfaces
    are repeats, so the de-duplication decides the inlier threshold, which must equal ll_register's bit for bit."""
    nc = M // 10
    ns = M - nc
    k = ns // 3
    corner = big.fc[:nc]
    surf = np.concatenate([big.fs[:ns - k], big.fs[:k]])
    check_dev_equals_register(big.ctx, big.m, corner, surf, state(big.guess))


def test_non_finite_features_next_to_the_sort_padding(big):
    """A non-finite surface feature's sort key equals the padding key in the bits the sort sees; only the stable sort keeps the real slots
    ahead of the padding.  NaN and +-inf surfaces in the last real slots, a NaN corner in the last corner slot, at several M below C."""
    T, C = big.T, big.C
    for M in (1000, 32 * T + 1, 256 * T + 1, C // 2, C - 1):
        nc = M // 10
        corner, surf = (a.copy() for a in big.feats(nc, M - nc))
        corner[-1, :3] = np.nan
        surf[-4, :3] = np.nan
        surf[-3, 0] = np.inf
        surf[-2, 1] = -np.inf
        surf[-1, 2] = np.nan
        check_dev_equals_register(big.ctx, big.m, corner, surf, state(big.guess))


def test_consecutive_calls_with_changing_splits(big):
    """One context in the order C, 1, 256T+1, 33, 512T+1, 32T+1, another in the reverse order: after launches where most CTAs returned early
    and after larger calls, every result equals ll_register and the other context's."""
    T, C = big.T, big.C
    order = [C, 1, 256 * T + 1, 33, 512 * T + 1, 32 * T + 1]
    st = state(big.guess)
    outs = []
    for seq in (order, order[::-1]):
        ctx, m = big.context(C)
        got = {}
        for M in seq:
            code, _, got[M] = check_dev_equals_register(ctx, m, *big.feats(M // 10, M - M // 10), st)
            got[M]["code"] = code
        outs.append(got)
        m.release(); ctx.close()
    assert outs[0] == outs[1]


@pytest.mark.parametrize("edge", ["256T+1", "512T+1"])
def test_deblur_past_one_tile(big, edge):
    """if_motion_deblur = 1 (the 56-byte slots) with two and three tiles per CTA; the feature intensities, the time stamps, span 0 ... 0.1."""
    M = EDGES[edge](big.T, big.C)
    corner, surf = big.feats(M // 10, M - M // 10)
    assert surf[:, 3].min() < 0.01 and surf[:, 3].max() > 0.09
    code, _, got = check_dev_equals_register(big.ctx, big.m, corner, surf, state(big.guess, if_motion_deblur=1))
    assert code == 0 and got["registered"] == 1


def test_max_features_rule_and_refusals(big):
    """nc + ns = max_features registers; one more is refused by the hand-over kernel's rule with ll_register's status and text, leaves the
    previous features, and the next call equals a fresh context's.  The hook refuses what ll_scan_to_pose would not run on device counts."""
    capi = _capi()
    from loam_livox_b200.registration import Context, Map
    C = big.C
    st = state(big.guess)
    ctx, m = big.context(C)
    check_dev_equals_register(ctx, m, *big.feats(C // 10, C - C // 10), st)
    before = last_features(ctx)
    over = big.feats(C // 2 + 1, C - C // 2)
    code, err, _ = dev_counts(ctx, m, *over, st)
    rcode, rerr, _ = register(ctx, m, *over, st)
    assert (code, err) == (rcode, rerr) == (capi.LL_ERR_CAPACITY, "more features than max_features")
    assert all(np.array_equal(x, y) for x, y in zip(last_features(ctx), before))
    none = np.zeros((0, 4), np.float32)
    assert check_dev_equals_register(ctx, m, none, none, st)[:2] == (capi.LL_ERR_NO_BLOCKS, "no features")
    nxt = big.feats(100, 900)
    after = check_dev_equals_register(ctx, m, *nxt, st)
    fresh, fm = big.context(C)
    alone = dev_counts(fresh, fm, *nxt, st)
    assert (alone[0], alone[2]) == (after[0], after[2])
    fm.release(); fresh.close()
    # refusals, before anything is enqueued
    too_many = np.zeros((C + 1, 4), np.float32)
    assert dev_counts(ctx, m, too_many, big.fs[:10], st)[:2] == (capi.LL_ERR_CAPACITY, "more corner or surface features than max_scan_points")
    assert dev_counts(ctx, m, big.fc[:10], too_many, st)[0] == capi.LL_ERR_CAPACITY
    refused = "ll_scan_to_pose would register on host-sized counts here"
    assert dev_counts(ctx, m, *nxt, state(big.guess, current_frame_index=10))[:2] == (capi.LL_ERR_INVALID, refused)   # the gate (:199)
    assert dev_counts(ctx, m, *nxt, state(big.guess, icp_max_iterations=0))[:2] == (capi.LL_ERR_INVALID, refused)
    m.release(); ctx.close()
    host = Context(0, max_scan_points=C, max_features=C - 1)   # max_features < max_scan_points: the host-sized path
    hm = Map(host, big.mc, big.ms)
    assert dev_counts(host, hm, *nxt, st)[:2] == (capi.LL_ERR_INVALID, refused)
    hm.release(); host.close()


def test_shared_memory_gate_between_deblur_and_plain(big):
    """max_features = max_scan_points = 13 x 256 T: 13 tiles per CTA fit the deblur slots (56 B, up to 14 tiles) but not the plain ones (64 B,
    up to 12).  The hook refuses plain and runs deblur; ll_scan_to_pose with deblur off takes the host-sized path, equals ll_register, and
    leaves the error text that was set before it."""
    capi = _capi()
    T = big.T
    cap = 13 * 256 * T
    assert solve_grid(T, cap) == (256, 13, T)
    ctx, m = big.context(cap)
    nxt = big.feats(1000, 9000)
    refused = "ll_scan_to_pose would register on host-sized counts here"
    assert dev_counts(ctx, m, *nxt, state(big.guess))[:2] == (capi.LL_ERR_INVALID, refused)
    for M in (256 * T + 1, 4 * 256 * T + 1):
        corner, surf = big.feats(M // 2, M - M // 2)
        code, _, got = check_dev_equals_register(ctx, m, corner, surf, state(big.guess, if_motion_deblur=1))
        assert code == 0 and got["registered"] == 1
    assert dev_counts(ctx, m, *nxt, state(big.guess))[:2] == (capi.LL_ERR_INVALID, refused)   # the error text before the call below
    pose = S.default_pose()
    code, err, got, nc, ns, (fc, fs) = call(ctx, m, S.make_scan(N, pose), 100.0, pipe(), state(big.guess))
    assert err == refused
    assert code == 0 and nc + ns > 1000
    assert (code, got) == register(ctx, m, fc, fs, state(big.guess))[::2]
    m.release(); ctx.close()


def test_real_scan_past_one_tile(big):
    """ll_scan_to_pose on a 100k-point scan with 1 cm leaves: the front end's counts give more than one tile per solver CTA."""
    pc = _capi().PipelineCfg(pieces=3, use_piece=0, extractor_leaf_corner=0.01, extractor_leaf_surf=0.01, mapping_leaf_corner=0.01,
                             mapping_leaf_surf=0.01, whole_frame=1)
    big.ctx._lib.ll_extract_reset(big.ctx.h)
    code, got, nc, ns = check_equals_register(big.ctx, big.m, S.make_scan(100000, big.pose), 100.0, pc, state(big.guess))
    assert nc + ns > 256 * big.T and code == 0 and got["registered"] == 1
