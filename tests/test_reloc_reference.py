"""The NumPy restatement of relocalization (tests/reloc_reference.py) against independent formulations, and the ctypes layout of ll_reloc_cfg /
ll_reloc_candidate against the header (no GPU)."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import scipy.ndimage as ndi

import reloc_reference as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("seed,r", [(0, 1), (1, 2), (2, 3), (3, 4), (4, 1)])
def test_dilation_is_a_cube_maximum_filter(seed, r):
    rng = np.random.default_rng(seed)
    occ = rng.random((7 + seed, 5 + 2 * seed, 11)) < 0.03
    occ[0, 0, 0] = True                       # a voxel on the border
    occ[-1, -1, -1] = True
    want = ndi.maximum_filter(occ.astype(np.uint8), size=2 * r + 1, mode="constant", cval=0).astype(bool)
    assert np.array_equal(R.dilate_separable(occ, r), want)
    assert np.array_equal(want, ndi.binary_dilation(occ, structure=np.ones((3, 3, 3), bool), iterations=r))


def test_pack_words_bit_order():
    g = np.zeros((2, 3, 7), bool)    # 42 voxels: two words
    g[0, 0, 0] = g[0, 1, 2] = g[1, 2, 6] = True
    w = R.pack_words(g)
    v = [0, 2 + 7 * 1, 6 + 7 * (2 + 3 * 1)]
    want = np.zeros(2, np.uint32)
    for x in v:
        want[x >> 5] |= np.uint32(1 << (x & 31))
    assert np.array_equal(w, want)


def test_index_cells_on_faces_and_negative_coordinates():
    res = 0.25
    pts = np.array([[-1.0, -2.0, -0.5, 0], [-0.75, -2.0, -0.5, 0], [0.5, 0.25, 1.0, 0], [np.nan, 0, 0, 0], [np.inf, 1, 1, 0]], np.float32)
    dims, lo, occ = R.occupancy([pts], res, 2)
    assert np.array_equal(lo, np.float32([-1.0, -2.0, -0.5]))
    # x: (0.5 - -1) / 0.25 = 6 exactly -> dims 6 + 1 + 4
    assert dims.tolist() == [11, 14, 11]
    c, ok = R.cells(pts[:3], lo, res, 2, dims)
    assert ok.all() and c[0].tolist() == [2, 2, 2] and c[1].tolist() == [3, 2, 2] and c[2].tolist() == [8, 11, 8]
    assert occ.sum() == 3


def test_scores_equal_a_plain_loop():
    rng = np.random.default_rng(5)
    clouds = [rng.uniform(-3, 3, (300, 4)).astype(np.float32), rng.uniform(-2, 4, (200, 4)).astype(np.float32)]
    dims, lo, g, _ = R.index(clouds, 0.5, 1)
    pts = rng.uniform(-2, 2, (40, 4)).astype(np.float32)
    pts[3, :3] = np.nan
    pts[4, :3] = 0.0
    pts[5, 0] = np.inf
    yaw = np.radians([0.0, 40.0, 200.0])
    rot = np.stack([np.cos(yaw / 2), 0 * yaw, 0 * yaw, np.sin(yaw / 2)], axis=1)
    t0, step, nt = (-4.0, -1.0, 0.0), (1.5, 0.7, 0.3), (6, 3, 2)
    a = R.scores(g, dims, lo, 0.5, 1, pts, rot, t0, step, nt)
    b = R.scores_loop(g, dims, lo, 0.5, 1, pts, rot, t0, step, nt)
    assert np.array_equal(a, b) and a.max() > a.min()


def vec_case(seed):
    """A small grid anchored at (-3, -2, -1.5) (res 0.5: voxel faces at exact multiples) and score points with non-finite ones, points on voxel
    faces and at negative coordinates; rotations with the identity, a 180 deg yaw (w = 0 exactly) and a tilted one."""
    rng = np.random.default_rng(seed)
    cloud = rng.uniform(-3, 3, (400, 4)).astype(np.float32)
    cloud[0, :3] = (-3.0, -2.0, -1.5)
    cloud[1, :3] = (3.0, 2.5, 1.5)
    pts = rng.uniform(-2.5, 2.5, (60, 4)).astype(np.float32)
    pts[:12, :3] = rng.integers(-8, 8, (12, 3)) * 0.25   # on voxel faces (and on them again after the lattice's steps of 0.5)
    pts[12, :3] = np.nan
    pts[13, 1] = np.inf
    pts[14, 2] = -np.inf
    pts[15, :3] = 0.0
    tilt = np.array([0.995, 0.05, -0.08, 0.02]); tilt /= np.linalg.norm(tilt)
    rot = np.array([[1.0, 0, 0, 0], [0.0, 0, 0, 1.0], tilt])
    return cloud, pts, rot


@pytest.mark.parametrize("t0,step,nt", [((-1.0, -0.5, 0.0), (0.5, 0.5, 0.5), (5, 3, 2)),     # steps landing every face on a face again
                                        ((0.3, 0.2, -0.1), (0.0, 0.0, 0.0), (3, 2, 2)),     # step 0: identical translations
                                        ((2.0, 1.0, 0.5), (-0.35, -0.5, -0.25), (7, 4, 3)),  # negative steps, points leaving the grid
                                        ((0.0, 0.0, 0.0), (1.0, 1.0, 1.0), (1, 1, 1))])
@pytest.mark.parametrize("chunk", [1, 2, 7, None])
def test_vectorised_scores_equal_the_per_hypothesis_scores_and_the_loop(t0, step, nt, chunk):
    cloud, pts, rot = vec_case(17)
    dims, lo, g, _ = R.index([cloud], 0.5, 1)
    a = R.scores_vec(g, dims, lo, 0.5, 1, pts, rot, t0, step, nt, chunk=chunk)
    b = R.scores(g, dims, lo, 0.5, 1, pts, rot, t0, step, nt)
    assert a.dtype == np.int32 and np.array_equal(a, b) and a.max() > 0
    if chunk == 1:
        assert np.array_equal(a, R.scores_loop(g, dims, lo, 0.5, 1, pts, rot, t0, step, nt))


def test_vectorised_scores_of_no_point_and_of_non_finite_points_only():
    cloud, pts, rot = vec_case(3)
    dims, lo, g, _ = R.index([cloud], 0.5, 0)
    for p in (pts[:0], pts[12:15]):
        assert np.array_equal(R.scores_vec(g, dims, lo, 0.5, 0, p, rot, (0, 0, 0), (0.5, 0.5, 0.5), (3, 2, 1)), np.zeros(18, np.int32))


def test_one_call_pipeline_is_scores_peaks_and_the_first_k():
    cloud, pts, rot = vec_case(5)
    dims, lo, g, _ = R.index([cloud[:150]], 0.5, 0)
    t0, step, nt = (-2.5, -2.0, 0.0), (0.6, 0.6, 0.5), (9, 9, 1)
    for K, cyclic in ((4, True), (16, False)):
        out = R.relocalize(g, dims, lo, 0.5, 0, pts, rot, t0, step, nt, K, cyclic=cyclic)
        sc = R.scores(g, dims, lo, 0.5, 0, pts, rot, t0, step, nt)
        hs, ss = R.peaks_brute(sc, 3, nt, cyclic)
        assert np.array_equal(out["scores"], sc) and out["n_peaks"] == hs.shape[0] > 4
        assert [(c["hypothesis"], c["score"]) for c in out["candidates"]] == list(zip(hs[:K].tolist(), ss[:K].tolist()))
        for c in out["candidates"]:
            q, t = R.candidate_pose(c["hypothesis"], rot, t0, step, nt)
            assert np.array_equal(c["q"], q) and np.array_equal(c["t"], t)


@pytest.mark.parametrize("n_rot", [1, 2, 3, 5])
@pytest.mark.parametrize("cyclic", [False, True])
def test_peaks_equal_a_brute_force_neighbourhood(n_rot, cyclic):
    rng = np.random.default_rng(10 * n_rot + cyclic)
    for nt in ((4, 3, 1), (1, 1, 1), (5, 1, 2), (3, 4, 3)):
        sc = rng.integers(0, 4, n_rot * int(np.prod(nt))).astype(np.int32)   # many ties
        h1, s1 = R.peaks(sc, n_rot, nt, cyclic)
        h2, s2 = R.peaks_brute(sc, n_rot, nt, cyclic)
        assert np.array_equal(h1, h2) and np.array_equal(s1, s2), (nt, sc)


def test_peaks_cyclic_wrap_decides():
    # rotation 0 and rotation 2 are neighbours only on a circle of 3
    sc = np.array([5, 0, 6], np.int32)
    assert R.peaks(sc, 3, (1, 1, 1), True)[0].tolist() == [2]
    assert R.peaks(sc, 3, (1, 1, 1), False)[0].tolist() == [2, 0]
    # a plateau: the lowest index wins
    assert R.peaks(np.array([3, 3, 3, 3], np.int32), 1, (4, 1, 1), False)[0].tolist() == [0]


def _header_struct(name):
    txt = open(os.path.join(ROOT, "include", "loamlivox_b200.h")).read()
    m = re.search(r"typedef struct \{(.*?)\} " + name + ";", txt, re.S)
    assert m, name
    body = re.sub(r"/\*.*?\*/", "", m.group(1), flags=re.S)
    return [ln.strip() for ln in body.split(";") if ln.strip()]


def test_ctypes_layout_matches_header():
    from loam_livox_b200 import capi
    decl = " ".join(_header_struct("ll_reloc_cfg"))
    names = [f for f, _ in capi.RelocCfg._fields_]
    assert names == ["n_rot", "rot_wxyz", "rot_cyclic", "t0", "step", "nt", "max_candidates"]
    pos = [re.search(r"[\s*]" + n + r"\b", decl).start() for n in names]
    assert pos == sorted(pos)
    assert C.sizeof(capi.RelocCfg) == 4 + 4 + 8 + 4 + 4 + 24 + 24 + 12 + 4
    assert capi.RelocCfg.t0.offset == 24 and capi.RelocCfg.nt.offset == 72 and capi.RelocCfg.max_candidates.offset == 84
    assert [f for f, _ in capi.RelocCandidate._fields_] == ["q_wxyz", "t", "score", "hypothesis"]
    assert C.sizeof(capi.RelocCandidate) == 64 and capi.RelocCandidate.score.offset == 56
    txt = open(os.path.join(ROOT, "include", "loamlivox_b200.h")).read()
    assert int(re.search(r"#define LL_RELOC_MAX_SCORE_POINTS (\d+)", txt).group(1)) == capi.LL_RELOC_MAX_SCORE_POINTS


def test_yaw_circle_and_window():
    from loam_livox_b200.registration import window_lattice, yaw_circle
    q = yaw_circle(10.0)
    assert q.shape == (36, 4) and np.allclose(np.linalg.norm(q, axis=1), 1.0)
    assert np.allclose(q[9], [np.cos(np.pi / 4), 0, 0, np.sin(np.pi / 4)])
    tilt = np.array([np.cos(0.05), np.sin(0.05), 0, 0])
    qt = yaw_circle(90.0, tilt)
    assert np.allclose(qt[0], tilt)
    t0, step, nt = window_lattice(((-1.0, 39.0, 1.0), (-5.0, 5.0, 1.0), (0.1, 0.1, 0.0)))
    assert nt == [41, 11, 1] and t0 == [-1.0, -5.0, 0.1]
