"""The device cell map (csrc/cellmap.cu, matching_mode 1) against oracle.CellMap, bit for bit, at its edges: cell faces, the range and FOV
boundaries of the assembly, the revisit threshold, store growth and table capacity, and the limits of the packed cell and voxel keys."""
import numpy as np
import pytest

from loam_livox_b200.capi import LoamLivoxError

pytestmark = pytest.mark.gpu
F = np.float32
QI = np.array([1.0, 0.0, 0.0, 0.0])


def _maps(ctx, oracle, resolution=1.0, revisit=2000, max_cells=0):
    from loam_livox_b200.registration import Points_cloud_map
    return Points_cloud_map(ctx, resolution, revisit, max_cells), oracle.CellMap(resolution, revisit)


def _pts(xyz):
    p = np.zeros((len(xyz), 4), F)
    p[:, :3] = np.asarray(xyz, F)
    return p


def _append(g, o, p):
    g.append_cloud(p)
    o.append_cloud(p)
    assert g.stats() == (o.cells(), o.points(), o.frame_idx())


def _assemble(g, o, q, t, rng, fov, leaf, replace=False):
    a, fa = g.assemble(q, t, rng, fov, leaf, replace)
    b, fb = o.assemble(q, t, rng, fov, leaf, replace)
    assert fa == fb and a.shape == b.shape and np.array_equal(a, b), (fa, fb, a.shape, b.shape)
    assert g.stats() == (o.cells(), o.points(), o.frame_idx())
    return a, fa


def _ulps(x):
    x = F(x)
    return [np.nextafter(x, F(-np.inf)), x, np.nextafter(x, F(np.inf))]


# ---------------------------------------------------------------------------------------------- cell faces
def test_cell_faces_all_octants(ctx, oracle):
    box = 0.5
    xyz = []
    for i in range(-4, 5):
        for v in _ulps(i * box) + _ulps(i * box + 0.25):            # faces (round-half-away ties of (p - 0.25) / 0.5) and centres
            for s in [(1, 1, 1), (-1, 1, 1), (1, -1, 1), (1, 1, -1), (-1, -1, 1), (-1, 1, -1), (1, -1, -1), (-1, -1, -1)]:
                xyz.append((s[0] * v, s[1] * v * F(0.5), s[2] * v * F(0.25)))
    xyz += [(-0.0, -0.0, -0.0), (-0.0, 0.0, 0.1), (0.0, -0.0, -0.1)]
    g, o = _maps(ctx, oracle)
    _append(g, o, _pts(xyz))
    _append(g, o, _pts(xyz[::-1]))
    for leaf in (0.1, 0.25, 0.5):
        _assemble(g, o, QI, np.array([-20.0, 0.0, 0.0]), 100.0, 80.0, leaf)


def test_cell_index_rounding_in_other_resolutions(ctx, oracle):
    rng = np.random.default_rng(8)
    for res in (0.02, 0.3, 1.0, 7.0):
        box = F(res * 0.5)
        i = rng.integers(-50, 50, 3000)
        v = (i.astype(F) * box)
        v = np.where(rng.random(3000) < 0.5, v, np.nextafter(v, F(np.inf) * np.sign(rng.random(3000) - 0.5)))
        p = _pts(np.stack([v, np.roll(v, 1), np.roll(v, 2)], 1))
        g, o = _maps(ctx, oracle, res)
        _append(g, o, p)
        _assemble(g, o, QI, np.array([-100.0 * res, 0.0, 0.0]), 1000.0, 89.0, float(box) / 4)


# ---------------------------------------------------------------------------------------------- assembly selection
def test_range_boundary_in_float_squared_norm(ctx, oracle):
    g, o = _maps(ctx, oracle)
    cells = [(0.25 + 0.5 * k, 0.25, 0.25) for k in range(0, 13)]
    _append(g, o, _pts(cells * 3))
    t = np.array([-2.75, 0.25, 0.25])                             # cell k centre at distance 3 + 0.5 k exactly
    for r in (3.0, 4.0, 5.5):
        for rr in _ulps(r):
            a, fa = _assemble(g, o, QI, t, float(rr), 45.0, 0.1)
            assert fa == int(round((r - 3.0) / 0.5)) + (1 if rr >= F(r) else 0), (r, rr, fa)


def test_fov_boundary_and_degenerate_directions(ctx, oracle):
    g, o = _maps(ctx, oracle)
    rng = np.random.default_rng(9)
    c = [(0.25 + 0.5 * i, 0.25 + 0.5 * j, 0.25 + 0.5 * k) for i in range(-4, 5) for j in range(-4, 5) for k in range(-2, 3)]
    _append(g, o, _pts(c) + _pts(rng.uniform(-0.2, 0.2, (len(c), 3))))
    for t in ([0.25, 0.25, 0.25], [-1.75, 0.25, 0.25], [0.25, -1.75, 0.25], [0.2500001, 0.25, 0.25], [0.24999999, 0.25, 0.25]):
        t = np.array(t)                                            # a centre at t (an == 0), on the axis (angle 0), at ax = 0 and ax = -tiny
        for fov in (0.0, -0.0, float(np.nextafter(F(0), F(1))), 45.0, 89.99, 90.0, 90.01, 180.0):
            _assemble(g, o, QI, t, 100.0, fov, 0.2)
    # angle 0 exactly: `0 * 57.3 < fov` is false at fov = 0 and true one float above
    t = np.array([-1.75, 0.25, 0.25])
    _, f0 = _assemble(g, o, QI, t, 100.0, 0.0, 0.2)
    _, f1 = _assemble(g, o, QI, t, 100.0, float(np.nextafter(F(0), F(1))), 0.2)
    assert f0 == 0 and f1 == 9                                      # the nine cells on the view axis (the first one's centre is t itself)
    q = np.array([np.cos(0.3), 0.0, 0.0, np.sin(0.3)])
    for fov in (10.0, 30.0, 60.0):
        _assemble(g, o, q, np.array([-0.3, 0.1, 0.0]), 3.0, fov, 0.2, replace=True)


# ---------------------------------------------------------------------------------------------- revisit
@pytest.mark.parametrize("threshold", [1, 2, 2000])
def test_revisit_thresholds(ctx, oracle, threshold):
    rng = np.random.default_rng(threshold)
    g, o = _maps(ctx, oracle, 1.0, threshold)
    a = _pts(rng.uniform(0, 2, (500, 3)))
    b = _pts(rng.uniform(10, 12, (500, 3)))
    stale = _pts(np.full((3000, 3), 0.3) + rng.uniform(-0.1, 0.1, (3000, 3)))
    seq = [a, b, b, stale, b, a[:10], np.concatenate([_pts([(30.3, 0.3, 0.3)]), _pts([(30.3, 0.3, 0.3)] * 5)]), b, b, b, a]
    for p in seq:
        _append(g, o, p)
    _assemble(g, o, QI, np.array([-5.0, 1.0, 1.0]), 100.0, 60.0, 0.1, replace=True)
    for p in (a, stale, b, b, a):                                      # revisits after a down-sample-and-replace
        _append(g, o, p)
    _assemble(g, o, QI, np.array([-5.0, 1.0, 1.0]), 100.0, 60.0, 0.1, replace=True)


def test_revisit_threshold_below_one_is_refused(ctx, oracle):
    from loam_livox_b200.registration import Points_cloud_map
    for thr in (0, -1):
        with pytest.raises(LoamLivoxError):
            Points_cloud_map(ctx, 1.0, thr)


# ---------------------------------------------------------------------------------------------- store and table
def test_store_grows_past_reservation_with_live_points(ctx, oracle):
    rng = np.random.default_rng(10)
    g, o = _maps(ctx, oracle)
    g.reserve(1000, 1000)
    _append(g, o, _pts(rng.normal(0, 3, (900, 3))))
    _append(g, o, _pts(rng.normal(0, 3, (150000, 3))))               # past the reservation: the store doubles and carries its points
    _assemble(g, o, QI, np.array([-8.0, 0.0, 0.0]), 100.0, 50.0, 0.2, replace=True)
    _append(g, o, _pts(rng.normal(0, 3, (70000, 3))))
    _assemble(g, o, QI, np.array([-8.0, 0.0, 0.0]), 100.0, 50.0, 0.2, replace=True)


def test_table_exactly_half_full_then_one_over(ctx, oracle):
    g, o = _maps(ctx, oracle, 1.0, 2000, max_cells=2048)               # table of 4096 slots
    c = [(0.25 + 0.5 * i, 0.25 + 0.5 * j, 0.25) for i in range(64) for j in range(32)]
    _append(g, o, _pts(c))
    assert g.stats()[0] == 2048
    _append(g, o, _pts(c[:100]))
    with pytest.raises(LoamLivoxError):
        g.append_cloud(_pts([(100.25, 0.25, 0.25)]))


def test_max_cells_above_2_29_is_refused(ctx):
    # the largest table has 2^30 slots (max_cells 2^29): beyond it, 2 x max_cells and the capacity would leave int
    import ctypes as C
    from loam_livox_b200 import capi
    for max_cells in (1 << 30, 2**31 - 1):
        h = C.c_void_p()
        assert ctx._lib.ll_cellmap_create(ctx.h, 1.0, 2000, max_cells, C.byref(h)) == capi.LL_ERR_INVALID and not h.value, max_cells


def test_many_points_in_one_voxel(ctx, oracle):
    rng = np.random.default_rng(11)
    g, o = _maps(ctx, oracle)
    p = _pts(F(0.31) + rng.uniform(0, 0.0099, (60000, 3)).astype(F))  # one voxel of 0.01: the centroid's float sum depends on the order
    p[::3, :3] *= F(1.0000001)
    _append(g, o, p)
    _append(g, o, p[::-1].copy())
    _assemble(g, o, QI, np.array([-5.0, 0.3, 0.3]), 100.0, 45.0, 0.01, replace=True)
    _assemble(g, o, QI, np.array([-5.0, 0.3, 0.3]), 100.0, 45.0, 0.01, replace=True)


# ---------------------------------------------------------------------------------------------- key limits
def test_voxel_leaf_limit(ctx, oracle):
    """Leaves down to cell / 512 are exact; finer ones are refused (PCL would pass a cell with an int32-overflowing voxel count through)."""
    rng = np.random.default_rng(12)
    g, o = _maps(ctx, oracle)
    flat = _pts(np.stack([rng.uniform(0.001, 0.499, 3000), rng.uniform(0.001, 0.499, 3000), np.full(3000, 0.3)], 1))
    spread = _pts(rng.uniform(0.501, 0.999, (3000, 3)))
    _append(g, o, flat)
    _append(g, o, spread)
    finest = F(0.5 / 512)
    assert float(F(0.5)) / float(finest) == 512.0
    _assemble(g, o, QI, np.array([-5.0, 0.5, 0.5]), 100.0, 60.0, float(finest))
    _assemble(g, o, QI, np.array([-5.0, 0.5, 0.5]), 100.0, 60.0, float(np.nextafter(finest, F(1))))
    for leaf in (float(np.nextafter(finest, F(0))), 2e-4, 5e-5):   # 5e-5: a flat cell of 10 000 leaves per axis; 2e-4: PCL passes the spread cell through
        with pytest.raises(LoamLivoxError):
            g.assemble(QI, np.array([-5.0, 0.5, 0.5]), 100.0, 60.0, leaf, False)
    _assemble(g, o, QI, np.array([-5.0, 0.5, 0.5]), 100.0, 60.0, float(finest), replace=True)


def test_cell_index_limits(ctx, oracle):
    box = 0.5
    lim = (1 << 20) - 1
    xyz = [(lim * box + 0.25, 0.25, 0.25), (-lim * box + 0.25, 0.25, 0.25), (0.25, lim * box + 0.25, -lim * box + 0.25),
           (0.25, 0.25, lim * box + 0.25), (-(lim + 1) * box + 0.25, 0.25, -(lim + 1) * box + 0.25), (0.25, 0.25, 0.25)]
    g, o = _maps(ctx, oracle)
    _append(g, o, _pts(xyz))
    assert g.stats()[0] == 6
    for t in ([lim * box - 5.0, 0.25, 0.25], [-(lim + 1) * box - 3.0, 0.25, -(lim + 1) * box + 0.25], [-5.0, 0.25, 0.25]):
        _assemble(g, o, QI, np.array(t), 50.0, 80.0, 0.1)
    over = [((lim + 1) * box + 0.25, 0.25, 0.25), (0.25, -(lim + 2) * box + 0.25, 0.25), (0.25, 0.25, 1e30), (0.3, 0.3, 0.3)]
    with pytest.raises(LoamLivoxError, match="cell index"):
        g.append_cloud(_pts(over))                                    # never aliased into another cell: the append reports them
    o.append_cloud(_pts(over[3:]))
    assert g.stats() == (o.cells(), o.points(), o.frame_idx())       # the in-range point went in, the frame index moved on
    _append(g, o, _pts([(0.3, 0.3, 0.3)]))                             # and the next append is clean
    _assemble(g, o, QI, np.array([-5.0, 0.25, 0.25]), 50.0, 80.0, 0.1)


def test_non_finite_points_are_dropped(ctx, oracle):
    rng = np.random.default_rng(13)
    p = _pts(rng.normal(0, 2, (5000, 3)))
    p[::37, 0] = np.nan
    p[3::41, 1] = np.inf
    p[5::43, 2] = -np.inf
    g, o = _maps(ctx, oracle)
    _append(g, o, p)
    _append(g, o, p[:1000])
    _assemble(g, o, QI, np.array([-6.0, 0.0, 0.0]), 100.0, 60.0, 0.2, replace=True)


def test_first_append_while_map_has_no_cell(ctx, oracle):
    g, o = _maps(ctx, oracle)
    _append(g, o, np.zeros((0, 4), F))
    _append(g, o, np.full((4, 4), np.nan, F))
    _append(g, o, _pts([(0.3, 0.3, 0.3)]))
    _append(g, o, _pts([(0.3, 0.3, 0.3)]))
    assert g.stats() == (1, 2, 7)
