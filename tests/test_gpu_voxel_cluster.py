"""VoxelGrid on one thread-block cluster (vg_cluster_chain_kernel, loam_livox_b200/csrc/cloud.cu) against the oracle, bit for bit.

Inputs whose host-known size is at most VG_CLUSTER_CAP points take the cluster path (one launch per call); larger ones the CUB passes.  Both
must give PCL's VoxelGrid exactly: bounds over the finite points, the int32 overflow gate (pass-through copies every input, in order), voxels
in ascending key order, every centroid a sequential fp32 sum in ascending input order.  Checked through ll_voxel_downsample (one VoxelGrid)
and through ll_scan_to_pose (the front end's two chains of two VoxelGrids, from device counts far below the scan size).
"""
import numpy as np
import pytest

from loam_livox_b200 import capi
from loam_livox_b200 import synthetic as S

pytestmark = pytest.mark.gpu

CAP = 16 * 6400   # VG_CLUSTER_CAP: VGC_CTAS x VGC_PER_CTA


def _vg(ctx, oracle, p, leaf):
    """Device VoxelGrid == oracle VoxelGrid bit for bit; returns (output, kernel launches of the call)."""
    from loam_livox_b200.registration import voxel_grid_filter
    p = np.ascontiguousarray(p, np.float32)
    l0 = ctx.launches()
    out = voxel_grid_filter(ctx, p, leaf)
    launches = ctx.launches() - l0
    ref = oracle.voxel_grid(p, leaf)
    assert out.shape == ref.shape and np.array_equal(out.view(np.uint32), ref.view(np.uint32))
    return out, launches


def _cloud(n, seed, lo=-3.0, hi=3.0):
    rng = np.random.default_rng(seed)
    p = rng.uniform(lo, hi, (n, 4)).astype(np.float32)
    p[:, 3] = rng.uniform(0, 255, n).astype(np.float32)
    return p


@pytest.mark.parametrize("n", [1, 2, 511, 12799, 12800, 12801, CAP - 1, CAP, CAP + 1])
def test_cluster_sizes_and_the_selection(ctx, oracle, n):
    """Sizes around one CTA's share and the capacity: up to CAP points one launch (the cluster), past it the CUB passes, same result."""
    out, launches = _vg(ctx, oracle, _cloud(n, n), 0.25)
    assert (launches == 1) == (n <= CAP), launches
    assert out.shape[0] <= n


def test_cluster_one_crowded_voxel(ctx, oracle):
    """100 000 points in one voxel: the sum runs over the positions of all eight CTAs, in input order (any other order rounds differently)."""
    p = _cloud(100000, 31, 0.001, 0.999)
    out, launches = _vg(ctx, oracle, p, 1.0)
    assert out.shape[0] == 1 and launches == 1


def test_cluster_runs_of_equal_keys_across_ctas(ctx, oracle):
    """Few voxels with thousands of points each: runs span CTA boundaries and radix digits repeat in every warp (the rank must be stable)."""
    rng = np.random.default_rng(32)
    p = _cloud(90000, 33, 0.0, 3.9)
    p = p[rng.permutation(p.shape[0])]
    out, _ = _vg(ctx, oracle, p, 1.0)
    assert out.shape[0] == 64


def test_cluster_all_nan_and_mixed_non_finite(ctx, oracle):
    """All-NaN: no output.  NaN / inf rows among finite ones: dropped, and they do not widen the bounds."""
    out, _ = _vg(ctx, oracle, np.full((50000, 4), np.nan, np.float32), 0.4)
    assert out.shape == (0, 4)
    rng = np.random.default_rng(34)
    p = _cloud(60000, 35)
    bad = rng.choice(p.shape[0], 3000, replace=False)
    p[bad[:1000], 0] = np.nan; p[bad[1000:2000], 1] = np.inf; p[bad[2000:], 2] = -np.inf
    _vg(ctx, oracle, p, 0.2)


@pytest.mark.parametrize("dims", [(256, 1, 1), (257, 1, 1), (256, 256, 1), (257, 256, 1), (256, 256, 256), (256, 256, 257)])
def test_cluster_keys_on_digit_boundaries(ctx, oracle, dims):
    """Grids whose largest key is just below / at a power of 256 (1 ... 4 radix passes), every corner voxel present."""
    rng = np.random.default_rng(sum(dims))
    n = 40000
    p = np.zeros((n, 4), np.float32)
    for k in range(3):
        p[:, k] = rng.integers(0, dims[k], n).astype(np.float32) + np.float32(0.5)
    p[:8, :3] = np.array([[(i >> k & 1) * (dims[k] - 1) + 0.5 for k in range(3)] for i in range(8)], np.float32)
    p[:, 3] = rng.uniform(0, 1, n)
    _vg(ctx, oracle, p[rng.permutation(n)], 1.0)


@pytest.mark.parametrize("n", [30000, CAP + 7])
def test_overflow_gate_both_sides_on_both_paths(ctx, oracle, n):
    """dx * dy * dz just below 2^31 - 1 (the grid is honoured) and just above (every input copied through in order, non-finite rows included)."""
    rng = np.random.default_rng(n)
    for dy, honoured in ((46340, True), (46341, False)):
        p = np.zeros((n, 4), np.float32)
        p[:, 0] = rng.integers(0, 46341, n); p[:, 1] = rng.integers(0, dy, n); p[:, 3] = rng.uniform(0, 1, n)
        p[:, :2] += np.float32(0.5)
        p[0, :2] = [0.0, 0.0]; p[1, :2] = [46340.5, dy - 0.5]
        p[2:40] = p[2]
        p[100:110, 0] = np.nan
        out, launches = _vg(ctx, oracle, p, 1.0)
        assert (launches == 1) == (n <= CAP)
        assert (out.shape[0] < n) == honoured
        if not honoured:
            assert np.array_equal(out.view(np.uint32), p.view(np.uint32))


@pytest.mark.parametrize("leaves", [(0.01, 0.01, 0.01, 0.02), (0.1, 0.2, 0.1, 0.4), (0.05, 0.05, 0.05, 0.1)])
def test_front_end_chains_match_the_oracle(oracle, leaves):
    """ll_scan_to_pose on a 100k-point scan: both chains start from device counts far below the scan size (about a thousand corners).  The
    first leaf set is bench.py's C2, where the surface chain's first VoxelGrid is a pass-through and its second a real one.  The features the
    registration used equal the oracle's chains bit for bit, and so do the counts."""
    from loam_livox_b200.registration import Context, Map, features_to_pointcloud2, scan_to_pose
    lc, ls, mlc, mls = leaves
    ctx = Context(0, max_scan_points=100000, max_features=100000)   # its own scan-time history, mirrored by one oracle extractor
    pose = S.default_pose()
    mc, ms = S.make_map(5000, 45000)
    raw = S.make_scan(100000, pose)
    m = Map(ctx, mc, ms)
    pc = capi.PipelineCfg(pieces=3, use_piece=0, extractor_leaf_corner=lc, extractor_leaf_surf=ls, mapping_leaf_corner=mlc, mapping_leaf_surf=mls, whole_frame=1)
    st = capi.default_reg_state(q_w_last=pose.q, t_w_last=pose.t, q_w_curr=pose.q, t_w_curr=pose.t)
    ex = oracle.Extractor()
    for _ in range(3):   # eager, captured, replayed front end
        _, nc, ns = scan_to_pose(ctx, m, raw, 100.0, pc, st)
        ex.extract(raw, 100.0)
        c, s, _ = ex.get_features(0.0, 1.0)
        c = oracle.voxel_grid(oracle.voxel_grid(c, lc), mlc)
        s = oracle.voxel_grid(oracle.voxel_grid(s, ls), mls)
        assert (nc, ns) == (c.shape[0], s.shape[0])
        for which, ref in ((0, c), (1, s)):
            got = np.frombuffer(features_to_pointcloud2(ctx, which), np.float32).reshape(-1, 4)
            assert np.array_equal(got.view(np.uint32), np.ascontiguousarray(ref, np.float32).view(np.uint32))
    m.release()
    ctx.close()
