"""GPU tests of three hot-path kernels at the edges the end-to-end scenes never reach, each against an exact reference:

- K10, the inlier threshold (compute_inlier_residual_threshold, point_cloud_registration.hpp:153-161), through ll_inlier_select: the fused solver
  kernel's grid-wide select, as the sharded mode runs it between its two solves, against NumPy;
- the kNN bucket tree (ll_knn) at the sizes where the tree changes shape and on degenerate geometry, against the oracle's brute force;
- VoxelGrid (ll_voxel_downsample) at voxel faces, the int32 overflow gate, large voxel populations and the block-size boundaries of its kernels,
  against the oracle and the independent NumPy restatement of tests/test_oracle.py.

Bars: exact (the threshold is one of the inputs; neighbour ids, fp32 distances and fp32 centroids are bit-exact elsewhere in the suite too).
"""
import ctypes as C

import numpy as np
import pytest

from loam_livox_b200 import capi
from loam_livox_b200 import synthetic as S
from test_oracle import K10_SIZES, _voxel_numpy, k10_vectors

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------- K10: inlier threshold
@pytest.mark.parametrize("n", K10_SIZES)
def test_inlier_select_matches_numpy(ctx, n):
    """Continuous values, all equal, ten values, signed zeros, runs of consecutive doubles that force every radix pass (bins of 64 / 65 values,
    the last pass), runs straddling a digit boundary, subnormals to 1e300, +inf / NaN slots; every ratio also at 1.0 (clamped to the last value)."""
    from loam_livox_b200.registration import inlier_select
    bad = []
    for name, v, ratios in k10_vectors(n):
        u = np.unique(v[np.isfinite(v)])
        for ratio in list(ratios) + [1.0]:
            want = u[min(int(ratio * len(u)), len(u) - 1)]
            got, nd = inlier_select(ctx, v, ratio)
            if not (nd == len(u) and got == want):
                bad.append((name, ratio, got, want, nd, len(u)))
    assert not bad, bad[:8]


def test_inlier_select_without_values_and_bad_arguments(ctx):
    from loam_livox_b200.registration import inlier_select
    for v in (np.zeros(0), np.array([np.inf, np.nan, np.inf]), np.full(5000, np.nan)):
        assert inlier_select(ctx, v, 0.8) == (0.0, 0)
    L, out, nd = capi.lib(), C.c_double(), C.c_int()
    big = np.ones(ctx.cfg.max_features + 1)
    assert L.ll_inlier_select(ctx.h, big.ctypes.data, big.shape[0], 0.8, C.byref(out), C.byref(nd)) == capi.LL_ERR_CAPACITY
    ok = np.ones(10)
    neg = np.array([1.0, -1.0])
    assert L.ll_inlier_select(ctx.h, neg.ctypes.data, 2, 0.8, C.byref(out), C.byref(nd)) == capi.LL_ERR_INVALID
    assert inlier_select(ctx, ok, 0.8) == (1.0, 1)   # the context is still usable


def _mk(nc, ns, qc, qs, seed=0):
    mc, ms = S.make_map(nc, ns, seed=S.SEED + seed)
    pose = S.default_pose()
    fc, fs = S.make_features(qc, qs, pose, seed=S.SEED + seed)
    return mc, ms, fc, fs, pose


def _register(ctx, m, fc, fs, guess, **kw):
    from loam_livox_b200.registration import Point_cloud_registration
    reg = Point_cloud_registration(ctx, **kw)
    reg.set_pose(guess.q, guess.t)
    st = reg.find_out_incremental_transfrom(m, fc, fs)
    r = reg.result
    return (st, r.icp_iterations, r.num_residual_blocks, r.total_lm_iterations, tuple(r.q_w_curr), tuple(r.t_w_curr), r.final_cost, r.inlier_threshold)


def test_inlier_select_keeps_the_solver_generation_protocol(oracle):
    """The hook kernel uses the solver's exchange rows: it must hand the advanced generation to the next launch, or a later registration on the same
    context could match a stale tag.  registration, hook, the same registration: both equal a fresh context's result bit for bit."""
    from loam_livox_b200.registration import Context, Map, inlier_select
    mc, ms, fc, fs, pose = _mk(500, 4500, 200, 1800)
    guess = S.perturb_pose(pose, np.random.default_rng(6))
    fresh = Context(0, max_scan_points=50000, max_features=50000)
    fm = Map(fresh, mc, ms)
    want = _register(fresh, fm, fc, fs, guess)
    fm.release()
    fresh.close()
    c = Context(0, max_scan_points=50000, max_features=50000)
    m = Map(c, mc, ms)
    assert _register(c, m, fc, fs, guess) == want
    v = np.random.default_rng(1).uniform(0, 1, 40000)
    for _ in range(3):   # several hook launches: each advances the generation by one exchange per radix pass + 2
        assert inlier_select(c, v, 0.8)[1] == 40000
    assert _register(c, m, fc, fs, guess) == want
    m.release()
    c.close()


# ---------------------------------------------------------------------------------------------- K10 end to end: duplicate L1 norms
@pytest.mark.parametrize("copies,cap", [(2, 1000000), (5, 1000000), (5, 200)])
def test_register_with_duplicate_features(ctx, oracle, copies, cap):
    """A third of the surface features repeated: identical blocks, exactly equal L1 norms; only the de-duplication of the std::set keeps the rank
    floor(ratio * n) right.  Against oracle.register: counts, ICP iterations, inlier threshold and pose."""
    from loam_livox_b200.registration import Map, Point_cloud_registration
    mc, ms, fc, fs, pose = _mk(5000, 45000, 1000, 9000)
    fs = np.concatenate([fs] + [fs[: fs.shape[0] // 3]] * (copies - 1))
    m = Map(ctx, mc, ms)
    guess = S.perturb_pose(pose, np.random.default_rng(copies))
    kw = dict(maximum_allow_residual_block=cap, rng_seed=copies)
    reg = Point_cloud_registration(ctx, **kw)
    reg.set_pose(guess.q, guess.t)
    st = reg.find_out_incremental_transfrom(m, fc, fs)
    p = oracle.default_params(q_w_last=guess.q, t_w_last=guess.t, q_w_curr=guess.q, t_w_curr=guess.t, **kw)
    ost, ores = oracle.register(mc, oracle.KdTree(mc), ms, oracle.KdTree(ms), fc, fs, p)
    r = reg.result
    assert st == ost == 1 and r.icp_iterations == ores.icp_iterations
    assert (r.corner_used, r.surf_used, r.num_residual_blocks) == (ores.corner_used, ores.surf_used, ores.num_residual_blocks)
    assert abs(r.inlier_threshold - ores.inlier_threshold) <= 1e-7 * ores.inlier_threshold
    dt = np.linalg.norm(np.array(r.t_w_curr) - np.array(ores.t_w_curr))
    da = S.quat_angle(np.array(r.q_w_curr), np.array(ores.q_w_curr))
    assert dt < 1e-7 and da < 1e-7, (dt, da)


# ---------------------------------------------------------------------------------------------- kNN bucket tree: shapes and geometry
def _knn_matches_brute(ctx, oracle, cloud, q):
    """5-NN of q in `cloud` (the surface index; the corner index gets the same cloud) against brute force, bit for bit; returns the answer."""
    from loam_livox_b200.registration import Map
    cloud = np.ascontiguousarray(cloud, np.float32)
    m = Map(ctx, cloud, cloud)
    idx, d2 = m.nearestKSearch(1, q)
    bi, bd, _ = oracle.knn_brute(cloud, q)
    fin = np.isfinite(q[:, :3]).all(1)
    assert np.array_equal(idx[fin], bi[fin]) and np.array_equal(d2[fin], bd[fin])
    assert (idx[~fin] == -1).all() and np.isposinf(d2[~fin]).all()   # a non-finite query has no neighbour: five -1 / +inf
    ci, cd = m.nearestKSearch(0, q)
    assert np.array_equal(ci, idx) and np.array_equal(cd, d2)
    m.release()
    return idx, d2


def _queries(rng, cloud, nq=256):
    pick = cloud[rng.integers(0, cloud.shape[0], nq)].copy()
    q = pick.copy()
    q[nq // 4:, :3] += rng.normal(0, 0.05, (nq - nq // 4, 3)).astype(np.float32)    # a quarter exactly on map points
    q[-8:, :3] = cloud[0, :3] + np.float32(1e4)                                     # far away
    q[-16:-8, :3] = np.array([0.0, -0.0, 0.0], np.float32)                          # +-0.0
    q[-17, :3] = [-0.0, -0.0, -0.0]
    q[-24:-17, :3] = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [np.nan] * 3, [np.inf] * 3, [1, np.nan, 1], [np.inf, -np.inf, np.nan]], np.float32)
    return q


@pytest.mark.parametrize("n", [1, 4, 5, 31, 32, 33, 1023, 1024, 1025, 32767, 32768, 32769])
def test_knn_at_tree_shape_boundaries(ctx, oracle, n):
    """A second bucket after 32 points, a second level after 1024 and a third after 32768, with partial nodes."""
    rng = np.random.default_rng(n)
    cloud = rng.normal(0, 5, (n, 4)).astype(np.float32)
    idx, _ = _knn_matches_brute(ctx, oracle, cloud, _queries(rng, cloud))
    assert (idx[:, min(n, 5):] == -1).all()


@pytest.mark.parametrize("copies", [5, 100, 5000])
def test_knn_all_points_identical(ctx, oracle, copies):
    rng = np.random.default_rng(copies)
    cloud = np.tile(np.array([[1.25, -3.5, 0.75, 7.0]], np.float32), (copies, 1))
    idx, d2 = _knn_matches_brute(ctx, oracle, cloud, _queries(rng, cloud))
    assert (idx[:64] == np.arange(5)).all() and (d2[:64] == 0).all()      # exact ties: the five smallest indices


def test_knn_degenerate_and_far_geometry(ctx, oracle):
    """Zero-extent axes of the Hilbert box (a plane z = 0 exactly, a line), two clusters 1e4 m apart, and a 5 cm blob at (1e5, -1e5, 50) where the
    fp32 spacing (7.8 mm) turns near points into exact duplicates."""
    rng = np.random.default_rng(11)
    plane = np.zeros((20000, 4), np.float32)
    plane[:, :2] = rng.uniform(-30, 30, (20000, 2))
    line = np.zeros((3000, 4), np.float32)
    line[:, 0] = rng.uniform(-10, 10, 3000)
    two = rng.normal(0, 1, (6000, 4)).astype(np.float32)
    two[3000:, :3] += np.float32(1e4)
    blob = (np.array([1e5, -1e5, 50.0]) + rng.uniform(-0.025, 0.025, (10000, 3))).astype(np.float32)
    blob = np.concatenate([blob, np.zeros((10000, 1), np.float32)], axis=1)
    assert np.unique(blob[:, 0]).shape[0] < 10 and np.unique(blob[:, 1]).shape[0] < 10
    for cloud in (plane, line, two, blob):
        _knn_matches_brute(ctx, oracle, cloud, _queries(rng, cloud))


def test_knn_ties_across_buckets(ctx, oracle):
    """100 copies of each of 50 points (copy c of point j at index 50 c + j): queries at the points get the 5 smallest indices, across buckets."""
    rng = np.random.default_rng(12)
    base = rng.uniform(-5, 5, (50, 4)).astype(np.float32)
    cloud = np.tile(base, (100, 1))
    q = np.concatenate([base, _queries(rng, cloud)])
    idx, d2 = _knn_matches_brute(ctx, oracle, cloud, q)
    assert np.array_equal(idx[:50], np.arange(50)[:, None] + 50 * np.arange(5)[None, :]) and (d2[:50] == 0).all()


def _blocks_match_oracle(ctx, oracle, mc, ms, fc, fs):
    """build_blocks against oracle.build_blocks as in test_gpu_parity.test_blocks_normal_equations_and_solve; a plane normal from coinciding
    neighbours is NaN on both sides (ceres_icp.hpp:329-332 divide by a zero norm)."""
    from loam_livox_b200.registration import Map, Point_cloud_registration
    m = Map(ctx, mc, ms)
    reg = Point_cloud_registration(ctx)
    reg.set_pose([1.0, 0, 0, 0], [0.0, 0, 0])
    typ, a3, v3, ca, sa = reg.build_blocks(m, fc, fs)
    p = oracle.default_params(q_w_last=[1.0, 0, 0, 0], t_w_last=[0.0, 0, 0], q_w_curr=[1.0, 0, 0, 0], t_w_curr=[0.0, 0, 0])
    blocks, src, oca, osa = oracle.build_blocks(mc, oracle.KdTree(mc), ms, oracle.KdTree(ms), fc, fs, p)
    assert (ca, sa) == (oca, osa)
    slot = src[:, 1] + np.where(src[:, 0] == 1, fc.shape[0], 0)
    assert np.array_equal(np.nonzero(typ)[0], slot)
    assert np.array_equal(typ[slot], blocks[:, 0].astype(np.int32) + 1)
    assert np.array_equal(a3[slot], blocks[:, 4:7])
    assert np.array_equal(np.isnan(v3[slot]), np.isnan(blocks[:, 7:10]))
    assert np.allclose(v3[slot], blocks[:, 7:10], rtol=0, atol=1e-15, equal_nan=True)
    m.release()
    return v3[slot]


def test_blocks_on_coplanar_map_and_on_duplicate_points(ctx, oracle):
    rng = np.random.default_rng(13)
    ms = np.zeros((20000, 4), np.float32)
    ms[:, :2] = rng.uniform(-20, 20, (20000, 2))                           # every point on z = 0 exactly
    mc = np.zeros((2000, 4), np.float32)
    mc[:, 0] = rng.uniform(-20, 20, 2000); mc[:, 2] = 1.0                  # one line
    fs = ms[rng.integers(0, 20000, 3000)].copy(); fs[:, 2] = rng.normal(0, 0.05, 3000).astype(np.float32)
    fc = mc[rng.integers(0, 2000, 300)].copy(); fc[:, 1:3] += rng.normal(0, 0.05, (300, 2)).astype(np.float32)
    v = _blocks_match_oracle(ctx, oracle, mc, ms, fc, fs)
    assert np.isfinite(v).all()
    dup = np.repeat(ms[:7000], 3, axis=0)                                   # each point three times: neighbours 0 / 2 can coincide
    dup[:, 2] = rng.normal(0, 0.02, 7000).repeat(3).astype(np.float32)
    v = _blocks_match_oracle(ctx, oracle, mc, dup, fc, fs)
    assert np.isnan(v).any()


# ---------------------------------------------------------------------------------------------- VoxelGrid
def _vg_matches(ctx, oracle, p, leaf, numpy=True):
    from loam_livox_b200.registration import voxel_grid_filter
    p = np.ascontiguousarray(p, np.float32)
    out = voxel_grid_filter(ctx, p, leaf)
    ref = oracle.voxel_grid(p, leaf)
    assert out.shape == ref.shape and np.array_equal(out.view(np.uint32), ref.view(np.uint32))
    if numpy:
        assert np.array_equal(out, _voxel_numpy(p, leaf))
    return out


def test_voxel_grid_one_crowded_voxel(ctx, oracle):
    """100 000 points in one voxel: one thread sums them in input order in fp32 (CentroidPoint), any other order rounds differently."""
    rng = np.random.default_rng(21)
    p = rng.uniform(0.001, 0.999, (100000, 4)).astype(np.float32)
    p[:, 3] = rng.uniform(0, 255, 100000).astype(np.float32)
    assert _vg_matches(ctx, oracle, p, 1.0).shape[0] == 1


@pytest.mark.parametrize("leaf", [0.25, 0.1])
def test_voxel_grid_points_on_faces_and_negative_coordinates(ctx, oracle, leaf):
    """Coordinates exactly on voxel faces (multiples of a representable leaf, and of 0.1 which is not), negative ones, -0.0 and -leaf."""
    rng = np.random.default_rng(22)
    lf = np.float32(leaf)
    ticks = np.concatenate([np.arange(-6, 7, dtype=np.float32) * lf, np.float32([-0.0, 0.0, -lf, lf, np.float32(-3) * lf])])
    g = np.stack(np.meshgrid(ticks, ticks, ticks, indexing="ij"), -1).reshape(-1, 3)
    p = np.concatenate([g, rng.uniform(0, 1, (g.shape[0], 1))], axis=1).astype(np.float32)
    p = np.concatenate([p, p[rng.integers(0, p.shape[0], 2000)]])            # repeated points: more than one per voxel
    _vg_matches(ctx, oracle, p[rng.permutation(p.shape[0])], leaf)


def test_voxel_grid_overflow_gate_both_sides(ctx, oracle):
    """dx * dy * dz just below 2^31 - 1 (46341 x 46340 x 1 voxels: the grid is honoured) and just above (46341 x 46341: PCL copies the input)."""
    rng = np.random.default_rng(23)
    for dy, honoured in ((46340, True), (46341, False)):
        p = np.zeros((3000, 4), np.float32)
        p[:, 0] = rng.integers(0, 46341, 3000); p[:, 1] = rng.integers(0, dy, 3000); p[:, 3] = rng.uniform(0, 1, 3000)
        p[:, :2] += np.float32(0.5)
        p[0, :2] = [0.0, 0.0]; p[1, :2] = [46340.5, dy - 0.5]                  # the box: (long long)(extent / 1.0) + 1 = 46341 and dy voxels
        p[2:40] = p[2]                                                       # one voxel with 38 points
        out = _vg_matches(ctx, oracle, p, 1.0, numpy=honoured)
        assert (out.shape[0] < p.shape[0]) == honoured and np.array_equal(out, p) != honoured


def test_voxel_grid_empty_and_all_nan(ctx, oracle):
    for p in (np.zeros((0, 4), np.float32), np.full((1000, 4), np.nan, np.float32)):
        assert _vg_matches(ctx, oracle, p, 0.4, numpy=False).shape == (0, 4)


@pytest.mark.parametrize("n", [1, 255, 256, 257, 67583, 67584, 67585, 3 * 67584 + 5])
def test_voxel_grid_block_boundaries(ctx, oracle, n):
    """256-thread blocks, and past 2 x 132 x 256 points vg_minmax_setup_kernel's capped grid: every thread loops over several points before the last
    block does the set-up."""
    rng = np.random.default_rng(n)
    p = rng.uniform(-3, 3, (n, 4)).astype(np.float32)
    p[n // 2, :3] = [3.5, -3.5, 3.5]                                         # the box corners sit in the middle of the input
    p[-1, :3] = [-3.5, 3.5, -3.5]
    _vg_matches(ctx, oracle, p, 0.5)
