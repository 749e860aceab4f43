"""The keyframe kernels on constructed inputs at their edges (keyframe_cases.py): cell typing, keyframe sizes, direction bins, ROI, blur and the
template search on the device, bit for bit against the keyframe oracle, and within stated tolerances of fp64 references."""
import numpy as np
import pytest

import keyframe_cases as KC
import keyframe_reference as K
from loam_livox_b200 import capi
from loam_livox_b200.registration import Keyframe, Points_cloud_map, loop_search

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cell_cases():
    return KC.cell_cases()


def _same(kf, o, ko, info):
    """The device keyframe equals the oracle's bit for bit: cells, types, vectors, info, the four images and the typed clouds."""
    oi = o.info(ko)
    keys, inc, typ, vec = kf.cells()
    okeys, oinc, otyp, ovec = o.cells(ko)
    assert np.array_equal(keys, okeys) and np.array_equal(inc, oinc)
    bad = np.flatnonzero((typ != otyp) | np.any(vec != ovec, axis=1))
    assert len(bad) == 0, (bad[:5], typ[bad[:5]], otyp[bad[:5]], vec[bad[:5]], ovec[bad[:5]])
    assert (info.cells, info.line_cells, info.plane_cells, info.accumulate_frames) == (oi["cells"], oi["line_cells"], oi["plane_cells"],
                                                                                     oi["accumulate_frames"])
    assert np.array_equal(np.array(info.center, np.float32), oi["center"]) and np.float32(info.roi_range) == oi["roi_range"]
    assert np.float32(info.ratio_nonzero_line) == oi["ratio_line"] and np.float32(info.ratio_nonzero_plane) == oi["ratio_plane"]
    imgs, oimgs = kf.images(), o.images(ko)
    assert np.array_equal(imgs, oimgs)   # counts and the blurred images: the device sums in the oracle's order
    for a in (0, 1):
        assert np.abs(imgs[2 + a] - K.fp64_blur(imgs[a])).max() <= 1e-6 * max(1.0, float(imgs[a].max()))
    for which in (capi.LL_CELL_LINE, capi.LL_CELL_PLANE, capi.LL_CELL_ALL):
        assert np.array_equal(kf.extract_specify_points(which), o.cloud(ko, which))
    return typ, vec


def _one_keyframe(ctx, cloud, incremental):
    """One append of cloud into a fresh map with one open keyframe, on the device and the oracle; both analyzed and compared."""
    g, o = Points_cloud_map(ctx, 1.0, 2147483647, 0), K.OracleMap(1.0, incremental=incremental)
    kf, ko = Keyframe(ctx), o.new_keyframe()
    Keyframe.append(ctx, g, np.c_[cloud, np.zeros(len(cloud))].astype(np.float32), [kf])
    o.append(cloud, [ko])
    o.analyze(ko)
    info = kf.analyze(g, incremental)
    typ, vec = _same(kf, o, ko, info)
    return kf, typ, vec, info


@pytest.mark.parametrize("incremental", [False, True])
@pytest.mark.parametrize("name", ["points_1_to_8", "one_third", "identical_points", "axis_aligned", "centre_gate", "far_cells", "big_cell"])
def test_cell_typing_at_its_edges(ctx, cell_cases, name, incremental):
    cells = cell_cases[name]
    kf, typ, vec, info = _one_keyframe(ctx, KC.cells_cloud(cells), incremental)
    keys = kf.cells()[0]
    order = {int(x): r for r, x in enumerate(keys)}
    B = 1 << 20
    checked = 0
    for (i, j, k), p, what in cells:
        r = order[((k + B) << 42) | ((j + B) << 21) | (i + B)]
        t, v, _, cov = K.cell_type(p, KC.centre(i, j, k), incremental=incremental)
        assert typ[r] == t and np.array_equal(vec[r], v), what
        # the eigenvector against NumPy's eigh (fp64) with the sign pinned, where the eigenvalue gap is large and the covariance symmetric (the
        # incremental recurrence's (2 d2) d1^T term is not: Jacobi reads its upper triangle, eigh its lower one)
        if t in (1, 2) and np.array_equal(cov, cov.T):
            w, V = np.linalg.eigh(cov.astype(np.float64))
            c = 0 if t == 2 else 2
            gap = min(abs(w[c] - w[x]) for x in range(3) if x != c) / max(abs(w).max(), 1e-30)
            if gap > 1e-3:
                e = V[:, c] * (1 if V[np.argmax(np.abs(V[:, c])), c] > 0 else -1)
                assert np.abs(vec[r] - e).max() <= 1e-6 / gap, (what, vec[r], e)
                checked += 1
    assert checked > 0 or incremental or name == "identical_points"


@pytest.mark.parametrize("n_cells", KC.SIZES)
def test_keyframe_sizes(ctx, n_cells):
    """C cells across the 128-thread typing block, the first growth of the cell list past 4096 and the bits of the cell sort."""
    for incremental in (False, True):
        _, _, _, info = _one_keyframe(ctx, KC.size_cloud(n_cells, seed=n_cells), incremental)
        assert info.cells == n_cells


@pytest.mark.parametrize("incremental", [False, True])
def test_keyframe_growing_past_4096_beside_an_open_one(ctx, incremental):
    """Keyframe 0 grows past 4096 cells over five appends while keyframe 1 is open for the last three; a cell revisited in every append is held
    in both incarnations, only the first of them incremental."""
    g, o = Points_cloud_map(ctx, 1.0, 2, 0), K.OracleMap(1.0, 2, incremental)
    kfs, oks = [Keyframe(ctx), Keyframe(ctx)], [o.new_keyframe(), o.new_keyframe()]
    for cloud, op in KC.growth_appends():
        Keyframe.append(ctx, g, np.c_[cloud, np.zeros(len(cloud))].astype(np.float32), [kfs[i] for i in op])
        o.append(cloud, [oks[i] for i in op])
    for kf, ko in zip(kfs, oks):
        o.analyze(ko)
        _same(kf, o, ko, kf.analyze(g, incremental))
    assert kfs[0].info().cells > 4096 and kfs[0].cells()[1].max() == 1


@pytest.mark.parametrize("name", list(KC.direction_cases()))
def test_direction_bins_at_their_edges(ctx, name):
    cloud, want_line, want_plane = KC.direction_cases()[name]
    kf, typ, vec, info = _one_keyframe(ctx, cloud, False)
    imgs = kf.images()
    assert np.array_equal(imgs[0], want_line) and np.array_equal(imgs[1], want_plane)
    cl, cp, _ = K.numpy_images(typ, vec)
    assert np.array_equal(imgs[0], cl) and np.array_equal(imgs[1], cp)
    assert np.float32(info.ratio_nonzero_line) == np.float32((want_line >= 1).sum()) / np.float32(3600)


@pytest.mark.parametrize("name", list(KC.roi_cases()))
def test_roi_range_at_its_edges(ctx, name):
    cloud = KC.roi_cases()[name]
    kf, _, _, info = _one_keyframe(ctx, cloud, False)
    keys = kf.cells()[0]
    B = 1 << 20
    ijk = np.c_[(keys & 0x1fffff).astype(np.int64) - B, ((keys >> 21) & 0x1fffff).astype(np.int64) - B, ((keys >> 42) & 0x1fffff).astype(np.int64) - B]
    c, roi = K.numpy_roi_range(np.array([KC.centre(*x) for x in ijk], np.float32))
    assert np.array_equal(np.array(info.center, np.float32), c) and np.float32(info.roi_range) == roi


def _search_keyframes(ctx, kfs_px):
    """One keyframe per (line pixels, plane cells), each in its own lattice cube of one map, device and oracle."""
    g, o = Points_cloud_map(ctx, 1.0, 2147483647, 0), K.OracleMap(1.0)
    kfs, oks = [], []
    for b, (px, planes) in enumerate(kfs_px):
        cloud = KC.pattern_cloud(px, planes, b + 1)
        kf, ko = Keyframe(ctx), o.new_keyframe()
        if len(cloud):
            Keyframe.append(ctx, g, np.c_[cloud, np.zeros(len(cloud))].astype(np.float32), [kf])
            o.append(cloud, [ko])
        o.analyze(ko)
        info = kf.analyze(g)
        if info.cells:
            _same(kf, o, ko, info)
        kfs.append(kf)
        oks.append(ko)
    return kfs, o, oks


@pytest.mark.parametrize("name", list(KC.search_cases()))
def test_search_at_its_edges(ctx, name):
    kfs_px = KC.search_cases()[name]
    kfs, o, oks = _search_keyframes(ctx, kfs_px)
    newest = len(kfs) - 1
    infos = [kf.info() for kf in kfs]
    cells = np.array([i.cells for i in infos], np.int64)
    roi = np.array([i.roi_range for i in infos], np.float32)
    rp = np.array([i.ratio_nonzero_plane for i in infos], np.float32)
    rl = np.array([i.ratio_nonzero_line for i in infos], np.float32)
    imgs = np.stack([np.stack([o.images(k)[3], o.images(k)[2]]) for k in oks])
    osims, _ = K.oracle_search(cells, roi, rp, rl, imgs, newest)
    loose = dict(K.DEFAULT_CFG, minimum_keyframe_differen=1, minimum_similarity_planar=0.5, plane_with_line=0.3, minimum_similarity_linear=0.3,
                 avail_ratio_plane=0.0, avail_ratio_line=0.0)
    for cfg in (K.DEFAULT_CFG, loose):
        sp, sl, cand = loop_search(ctx, kfs, newest, capi.default_loop_cfg(**cfg))
        assert np.array_equal(sp, osims[:, 0]) and np.array_equal(sl, osims[:, 1])
        assert cand == K.numpy_gates(cells, roi, rp, rl, np.c_[sp, sl], newest, cfg) == K.oracle_gates(cells, roi, rp, rl, osims, newest, cfg)
    for his in range(newest) if newest < 20 else (0, newest - 1):
        for w, s in ((0, sp[his]), (1, sl[his])):
            assert abs(float(s) - K.fp64_similarity(imgs[newest, w], imgs[his, w])) <= 2e-6
    line_px = kfs_px[-1][0]
    for his, (px, planes) in enumerate(kfs_px[:-1]):
        shifted = newest < 20 and px and len(px) == len(line_px) and any(px == KC.roll(line_px, dp, dt) for dp in range(60) for dt in range(60))
        if shifted or (his == 0 and name == "newest_300" and px):   # a cyclic shift of the newest's line image (any shift: the wrap pad reaches every offset) scores exactly 1
            assert sl[his] == 1.0, his
        if planes and kfs_px[-1][1]:   # one-pixel plane images at the same pixel
            assert sp[his] == 1.0
        if not px or not line_px:   # an all-zero template or image
            assert sl[his] == 0.0
    if name == "cyclic_shifts":
        assert (sl[:-1] == 1.0).all() and sl[-1] < 1.0   # every shift, 31 included, scores 1; one pixel more does not


def test_blur_of_a_cyclic_shift_is_the_shifted_blur(ctx):
    base = KC.search_cases()["newest_1"][0][0]
    shifts = [(0, 0), (1, 0), (0, 59), (30, 30), (-13, 29)]
    kfs, _, _ = _search_keyframes(ctx, [(KC.roll(base, *s), 0) for s in shifts])
    ref = kfs[0].images()
    for kf, s in zip(kfs[1:], shifts[1:]):
        im = kf.images()
        assert np.array_equal(im[0], np.roll(ref[0], s, (0, 1))) and np.array_equal(im[2], np.roll(ref[2], s, (0, 1)))
