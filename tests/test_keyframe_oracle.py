"""The keyframe oracle (oracle/orc_keyframe.hpp) against real OpenCV, NumPy and its own restated gates, on the CPU."""
import ctypes as C

import cv2
import numpy as np
import pytest

import keyframe_reference as K

RNG = np.random.default_rng(7)


def _images():
    z = np.zeros((60, 60), np.float32)
    rnd = RNG.random((60, 60)).astype(np.float32) * 5
    sparse = np.zeros((60, 60), np.float32)
    idx = RNG.integers(0, 60, size=(40, 2))
    for i, j in idx:
        sparse[i, j] += 1
    one = np.zeros((60, 60), np.float32)
    one[0, 59] = 3
    return {"zero": z, "random": rnd, "sparse": sparse, "corner": one}


def test_gaussian_kernel_is_opencvs():
    assert np.array_equal(K.gaussian_kernel(), cv2.getGaussianKernel(9, 4, ktype=cv2.CV_32F).ravel())


@pytest.mark.parametrize("name", ["zero", "random", "sparse", "corner"])
def test_blur_equals_opencv(name):
    img = _images()[name]
    padded = np.pad(img, 5, mode="wrap")
    ref = cv2.GaussianBlur(padded, (9, 9), 4)[5:65, 5:65]
    got = K.blur(img)
    # OpenCV's separable filter sums the symmetric taps in pairs; the oracle in tap order: a few float ulps of the largest value
    assert np.abs(got - ref).max() <= 4e-7 * max(1.0, float(img.max())), np.abs(got - ref).max()


@pytest.mark.parametrize("pair", [("random", "random"), ("sparse", "random"), ("sparse", "sparse"), ("corner", "sparse"), ("zero", "sparse"),
                                  ("sparse", "zero"), ("zero", "zero")])
def test_similarity_equals_opencv_match_template(pair):
    imgs = _images()
    a, b = K.blur(imgs[pair[0]]), K.blur(RNG.permutation(imgs[pair[1]]).astype(np.float32))
    res = cv2.matchTemplate(np.pad(b, 30, mode="wrap"), a, cv2.TM_CCORR_NORMED)
    assert res.shape == (61, 61)
    got = K.similarity(a, b)
    # CCORR_NORMED at a zero norm (an all-zero template or image window) is 0 in OpenCV and in the oracle
    if not a.any() or not b.any():
        assert got == 0.0 and res.max() == 0.0
    else:
        assert abs(got - float(res.max())) <= 1e-5, (got, res.max())


def test_similarity_of_an_image_with_itself_is_one():
    a = K.blur(_images()["sparse"])
    assert abs(K.similarity(a, a) - 1.0) <= 1e-6


@pytest.mark.parametrize("seed", range(6))
def test_eig3_equals_numpy_eigh_up_to_the_pinned_sign(seed):
    r = np.random.default_rng(seed)
    B = r.normal(size=(3, 3)) * (10.0 ** r.integers(-3, 3))
    A = B @ B.T if seed % 2 else np.diag(r.random(3))
    w, V = K.eig3(A)
    wn, Vn = np.linalg.eigh(A)
    assert np.allclose(w, wn, rtol=1e-12, atol=1e-14 * np.abs(wn).max())
    for c in range(3):
        v = Vn[:, c] * (1 if Vn[np.argmax(np.abs(Vn[:, c])), c] > 0 else -1)
        assert np.allclose(V[:, c], v, atol=1e-9)
        assert V[np.argmax(np.abs(V[:, c])), c] > 0
    assert np.allclose(V @ np.diag(w) @ V.T, A, atol=1e-12 * max(1.0, np.abs(A).max()))


def _cell(kind, n=50, seed=0):
    r = np.random.default_rng(seed)
    if kind == "plane":
        p = np.c_[r.uniform(-0.2, 0.2, n), r.uniform(-0.2, 0.2, n), r.normal(0, 0.002, n)]
    elif kind == "line":
        p = np.c_[r.uniform(-0.2, 0.2, n), r.normal(0, 0.002, n), r.normal(0, 0.002, n)]
    else:
        p = r.normal(0, 0.1, (n, 3))
    return (p + 0.25).astype(np.float32)


@pytest.mark.parametrize("incremental", [False, True])
def test_typing_of_constructed_cells(incremental):
    c = np.array([0.25, 0.25, 0.25], np.float32)
    t, v, _, _ = K.cell_type(_cell("plane"), c, incremental=incremental)
    assert t == K_PLANE and abs(abs(v[2]) - 1) < 1e-3
    t, v, _, _ = K.cell_type(_cell("line"), c, incremental=incremental)
    assert t == K_LINE and abs(abs(v[0]) - 1) < 1e-3
    assert K.cell_type(_cell("blob"), c, incremental=incremental)[0] == K_SPHERE
    assert K.cell_type(_cell("plane", 4), c, incremental=incremental)[0] == K_SPHERE   # fewer than 5 points
    assert K.cell_type(_cell("plane", 5), c, incremental=incremental)[0] == K_PLANE
    # mean more than 0.75 res from the centre
    assert K.cell_type(_cell("plane") + np.float32(0.4), c, incremental=incremental)[0] == K_SPHERE
    assert K.cell_type(_cell("plane") + np.float32(0.2), c, incremental=incremental)[0] == K_PLANE


K_SPHERE, K_LINE, K_PLANE = 0, 1, 2


def test_batch_covariance_equals_numpy_with_n_minus_1():
    p = _cell("blob", 40, 3)
    _, _, mean, cov = K.cell_type(p, np.array([0.25, 0.25, 0.25], np.float32))
    assert np.allclose(mean, p.astype(np.float64).mean(0), atol=1e-6)
    assert np.allclose(cov, np.cov(p.astype(np.float64).T, ddof=1), atol=1e-6)


def test_incremental_covariance_tracks_the_batch_one():
    p = _cell("plane", 200, 4)
    _, _, _, ci = K.cell_type(p, np.array([0.25, 0.25, 0.25], np.float32), incremental=True)
    _, _, _, cb = K.cell_type(p, np.array([0.25, 0.25, 0.25], np.float32), incremental=False)
    # the recurrence starts from the 4-point covariance (append_pt's get_covmat skips 5 and 6 points), so it is not the batch one
    assert not np.array_equal(ci, cb)
    assert np.allclose(ci, cb, atol=2e-3)


def test_typing_follows_the_one_third_rule_at_one_ulp():
    """Six points on the axes (mean exactly 0, diagonal covariance): stepping the z extent one float at a time moves l1 / 3 across l0."""
    flips = 0
    last = None
    z = np.float32(np.sqrt((np.float32(0.004) / 3) * 5 / 2))   # 2 z^2 / 5 = l1 / 3 with l1 = 2 * 0.1^2 / 5
    for _ in range(300):
        z = np.nextafter(z, np.float32(0), dtype=np.float32)
    for _ in range(600):
        pts = np.array([[0.2, 0, 0], [-0.2, 0, 0], [0, 0.1, 0], [0, -0.1, 0], [0, 0, z], [0, 0, -z]], np.float32)
        t, _, _, cov = K.cell_type(pts, np.zeros(3, np.float32))
        w = np.sort(np.diag(cov).astype(np.float64))
        want = K_PLANE if w[1] * (1.0 / 3.0) > w[0] else (K_LINE if w[2] * (1.0 / 3.0) > w[1] else K_SPHERE)
        assert t == want
        if last is not None and t != last:
            flips += 1
        last = t
        z = np.nextafter(z, np.float32(1), dtype=np.float32)
    assert flips >= 1


def test_gates_equal_numpy_restatement():
    r = np.random.default_rng(11)
    n = 300
    for trial in range(20):
        cells = r.integers(0, 4000, n)
        roi = r.uniform(5, 15, n).astype(np.float32)
        rp, rl = r.uniform(0, 0.1, n).astype(np.float32), r.uniform(0, 0.06, n).astype(np.float32)
        sims = r.uniform(0.5, 1.0, (n, 2)).astype(np.float32)
        newest = n - 1 - trial
        cfg = dict(K.DEFAULT_CFG, minimum_keyframe_differen=int(r.integers(0, 250)))
        assert K.oracle_gates(cells, roi, rp, rl, sims, newest, cfg) == K.numpy_gates(cells, roi, rp, rl, sims, newest, cfg)


def test_gate_edges():
    newest = 4
    cells = np.array([100, 100, 100, 100, 100])
    roi = np.full(5, 10.0, np.float32)
    rp, rl = np.full(5, 0.1, np.float32), np.full(5, 0.1, np.float32)
    sims = np.full((5, 2), 0.99, np.float32)
    cfg = dict(K.DEFAULT_CFG, minimum_keyframe_differen=3)

    def both(*a, c=cfg):
        o = K.oracle_gates(*a, newest, c)
        assert o == K.numpy_gates(*a, newest, c)
        return o
    # his exactly minimum_keyframe_differen apart (5 - 2 = 3) passes, 5 - 3 = 2 does not
    assert both(cells, roi, rp, rl, sims) == [0, 1, 2]
    # the nonzero-ratio gate needs both below
    rp2, rl2 = rp.copy(), rl.copy(); rp2[0] = 0.04; rl2[0] = 0.02; rp2[1] = 0.04
    assert both(cells, roi, rp2, rl2, sims) == [1, 2]
    # ROI: |d| = 5 passes, one float more does not (std::abs on a float)
    roi2 = roi.copy(); roi2[0] = 15.0; roi2[1] = np.nextafter(np.float32(15.0), np.float32(20))
    assert both(cells, roi2, rp, rl, sims) == [0, 2]
    # similarities: plane > 0.94 alone, or line > 0.65 with plane > 0.92 (a double: the float 0.92f = 0.92000001669 passes it)
    s2 = sims.copy(); s2[0] = (0.94, 0.1); s2[1] = (0.93, 0.66); s2[2] = (0.92, 0.9)
    assert both(cells, roi, rp, rl, s2) == [1, 2]
    s2[2] = (np.nextafter(np.float32(0.92), np.float32(0)), 0.9)
    assert both(cells, roi, rp, rl, s2) == [1]
    # cell counts in size_t: a pair passes only when the newest has at least as many cells and the other has some
    c2 = cells.copy(); c2[0] = 101; c2[1] = 0; c2[2] = 99
    assert both(c2, roi, rp, rl, sims) == [2]
    c3 = np.zeros(5, np.int64)
    assert both(c3, roi, rp, rl, sims) == []


def test_oracle_roi_range_and_images_match_numpy():
    r = np.random.default_rng(5)
    m = K.OracleMap(1.0)
    k = m.new_keyframe()
    # a room corner: two walls and a floor, plus poles
    pts = []
    pts.append(np.c_[r.uniform(0, 8, 20000), r.uniform(0, 6, 20000), r.normal(0, 0.01, 20000)])
    pts.append(np.c_[r.normal(0, 0.01, 10000), r.uniform(0, 6, 10000), r.uniform(0, 3, 10000)])
    pts.append(np.c_[r.uniform(0, 8, 10000), r.normal(6, 0.01, 10000), r.uniform(0, 3, 10000)])
    for px in (2.1, 4.3, 6.2):
        pts.append(np.c_[r.normal(px, 0.01, 3000), r.normal(3.1, 0.01, 3000), r.uniform(0, 3, 3000)])
    m.append(np.vstack(pts), [k])
    m.analyze(k)
    info = m.info(k)
    keys, inc, typ, vec = m.cells(k)
    assert info["line_cells"] > 10 and info["plane_cells"] > 100
    B = 1 << 20
    ijk = np.c_[(keys & 0x1fffff).astype(np.int64) - B, ((keys >> 21) & 0x1fffff).astype(np.int64) - B, ((keys >> 42) & 0x1fffff).astype(np.int64) - B]
    centers = (ijk.astype(np.float32) * np.float32(0.5) + np.float32(0.25)).astype(np.float32)
    c, roi = K.numpy_roi_range(centers)
    assert np.array_equal(c, info["center"]) and roi == info["roi_range"]
    imgs = m.images(k)
    cnt_line, cnt_plane, _ = K.numpy_images(typ, vec)
    for cnt, idx, ratio in ((cnt_line, 0, info["ratio_line"]), (cnt_plane, 1, info["ratio_plane"])):
        assert np.array_equal(cnt, imgs[idx])
        assert np.float32((cnt >= 1).sum()) / np.float32(3600) == ratio
        assert np.array_equal(K.blur(cnt), imgs[2 + idx])


def test_keyframe_cell_sets_follow_append_cloud():
    m = K.OracleMap(1.0, revisit_threshold=2)
    a, b = m.new_keyframe(), m.new_keyframe()
    base = np.array([[0.1, 0.1, 0.1]], np.float32)
    # first append: every touched cell, also with one point
    m.append(np.vstack([base, base + 1, base + 1]), [a])
    assert m.info(a)["cells"] == 2
    # afterwards 3 points make a cell join, 2 do not
    m.append(np.vstack([base + 2] * 2 + [base + 3] * 3 + [base + 4] * 4), [a, b])
    assert m.info(b)["cells"] == 2 and m.info(a)["cells"] == 4 and m.info(a)["accumulate_frames"] == 2
    # a revisit past the threshold: a new incarnation of cell 0 joins b, a keeps the old one too when it gets it again
    m.append(np.vstack([base] * 3), [a, b])
    m.append(np.vstack([base] * 3), [a, b])
    keys, inc, _, _ = m.cells(a)
    assert sorted(inc.tolist()).count(1) == 1 and len(keys) == 5


def test_cabi_declares_the_loop_detection_entry_points():
    from loam_livox_b200 import capi
    L = C.CDLL(capi.LIB_PATH)
    for n in ("ll_keyframe_create", "ll_keyframe_append", "ll_keyframe_analyze", "ll_keyframe_images", "ll_keyframe_cloud", "ll_keyframe_cells",
              "ll_loop_search", "ll_loop_cfg_default", "ll_keyframe_get_info", "ll_keyframe_release"):
        assert n in capi.EXPORTS and hasattr(L, n)
    cfg = capi.default_loop_cfg()
    got = {f: getattr(cfg, f) for f, _ in capi.LoopCfg._fields_}
    assert got["minimum_keyframe_differen"] == 200
    for k in ("avail_ratio_plane", "avail_ratio_line", "maximum_roi_difference", "minimum_similarity_linear", "minimum_similarity_planar"):
        assert np.float32(got[k]) == np.float32(K.DEFAULT_CFG[k])
    assert got["plane_with_line"] == 0.92   # the double literal of laser_mapping.hpp:1012
    assert C.sizeof(capi.KeyframeInfo) == 4 * 4 + 6 * 4 + 3 * 8


def test_cpp_mirror_compiles_links_and_runs(tmp_path):
    import os
    import subprocess
    from loam_livox_b200 import capi
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "keyframe_mirror")
    libdir = os.path.dirname(capi.LIB_PATH)
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(root, "include"), os.path.join(root, "tests", "cpp", "keyframe_mirror.cpp"), "-o", exe,
           "-L", libdir, "-lloamlivox_b200", "-L", "/usr/local/cuda/lib64", "-lcudart", f"-Wl,-rpath,{libdir}", "-Wl,-rpath,/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "GPU run" in r.stdout or "no GPU" in r.stdout


def test_fp32_against_fp64_typing_on_a_scene():
    """The cells are typed from the float covariance by an fp64 eigen-decomposition; the reference decomposes in float (COMP_TYPE).  On a noisy
    room-corner scene, count the cells whose type changes when the eigenvalues come from a float32 solver (LAPACK ssyevd through NumPy)."""
    r = np.random.default_rng(21)
    n = 40000
    p = np.vstack([np.c_[r.uniform(0, 8, n), r.uniform(0, 6, n), r.normal(0, 0.03, n)],
                   np.c_[r.normal(0, 0.03, n // 2), r.uniform(0, 6, n // 2), r.uniform(0, 3, n // 2)],
                   np.c_[r.normal(3, 0.05, n // 4), r.normal(3, 0.05, n // 4), r.uniform(0, 3, n // 4)],
                   r.uniform(0, 8, (n // 4, 3))]).astype(np.float32)
    key = np.round((p - np.float32(0.25)) / np.float32(0.5)).astype(np.int64)
    order = np.lexsort((key[:, 0], key[:, 1], key[:, 2]))
    kp, pp = key[order], p[order]
    cuts = np.flatnonzero(np.any(np.diff(kp, axis=0) != 0, axis=1)) + 1
    typed = differ = 0
    for idx, cell in zip(np.split(np.arange(len(pp)), cuts), np.split(pp, cuts)):
        if len(cell) < 5:
            continue
        centre = (kp[idx[0]].astype(np.float32) * np.float32(0.5) + np.float32(0.25)).astype(np.float32)
        t, _, _, cov = K.cell_type(cell, centre)
        mean = cell.astype(np.float64).mean(0)
        if np.linalg.norm(mean - centre) > 0.375:
            continue
        typed += 1
        w = np.linalg.eigvalsh(cov.astype(np.float32)).astype(np.float64)
        t32 = K_PLANE if w[1] * (1.0 / 3.0) > w[0] else (K_LINE if w[2] * (1.0 / 3.0) > w[1] else K_SPHERE)
        differ += t32 != t
    print(f"fp32 vs fp64 typing: {differ} of {typed} cells differ")
    assert typed > 500 and differ <= 0.01 * typed


# ---- the constructed edge cases (keyframe_cases.py): each reaches its edge, and the oracle equals the NumPy and fp64 references on it --------
import keyframe_cases as KC   # noqa: E402


def _oracle_keyframe(cloud, incremental=False):
    m = K.OracleMap(1.0, incremental=incremental)
    k = m.new_keyframe()
    m.append(cloud, [k])
    m.analyze(k)
    return m, k


def _key(ijk):
    B = 1 << 20
    i, j, k = ijk
    return np.uint64(((k + B) << 42) | ((j + B) << 21) | (i + B))


def _fp64_type(p, c):
    """determine_feature on the exact (fp64) mean and covariance."""
    p = np.asarray(p, np.float64)
    if len(p) < 5 or np.linalg.norm(c - p.mean(0)) > 0.375:
        return K_SPHERE
    w = np.linalg.eigvalsh(np.cov(p.T, ddof=1))
    return K_PLANE if w[1] / 3 > w[0] else (K_LINE if w[2] / 3 > w[1] else K_SPHERE)


@pytest.mark.parametrize("name", list(KC.cell_cases()))
def test_cell_cases_oracle_equals_the_references(name):
    """Every cell lies in its designed map cell; the keyframe's types and vectors are those of the one-cell oracle (Points_cloud_cell) on its
    points, batch and incremental; the images, centre and ROI equal the NumPy restatements, the blur the fp64 one."""
    cells = KC.cell_cases()[name]
    for ijk, p, what in cells:
        assert (KC.cell_of(p) == np.array(ijk)).all(), what
    for inc in (False, True):
        m, k = _oracle_keyframe(KC.cells_cloud(cells), inc)
        keys, _, typ, vec = m.cells(k)
        order = {int(x): r for r, x in enumerate(keys)}
        assert len(order) == len(cells)
        for ijk, p, what in cells:
            t, v, _, _ = K.cell_type(p, KC.centre(*ijk), incremental=inc)
            r = order[int(_key(ijk))]
            assert typ[r] == t and np.array_equal(vec[r], v), (what, inc)
        info, imgs = m.info(k), m.images(k)
        cl, cp, _ = K.numpy_images(typ, vec)
        assert np.array_equal(imgs[0], cl) and np.array_equal(imgs[1], cp)
        centres = np.array([KC.centre(*ijk) for ijk, _, _ in sorted(cells, key=lambda c: int(_key(c[0])))], np.float32)
        c, roi = K.numpy_roi_range(centres)
        assert np.array_equal(c, info["center"]) and roi == info["roi_range"]
        for a in (0, 1):
            assert np.abs(imgs[2 + a] - K.fp64_blur(imgs[a])).max() <= 1e-6 * max(1.0, float(imgs[a].max()))


def test_cell_cases_reach_their_edges():
    cc = KC.cell_cases()
    get = {(name, what): (ijk, p) for name, cells in cc.items() for ijk, p, what in cells}

    def typed(name, what, inc=False):
        ijk, p = get[(name, what)]
        return K.cell_type(p, KC.centre(*ijk), incremental=inc)
    # incremental: 5 and 6 points keep the 4-point covariance, the 7th starts the recurrence
    for rep in range(3):
        ijk, p = [(c[0], c[1]) for c in cc["points_1_to_8"] if c[0] == (8, rep, 0)][0]
        c4 = K.cell_type(p[:4], KC.centre(*ijk), incremental=True)[3]
        for n, same in ((5, True), (6, True), (7, False)):
            assert np.array_equal(K.cell_type(p[:n], KC.centre(*ijk), incremental=True)[3], c4) == same
    # exact ties of the one-third rule: w1 = 3 w0 types LINE (not PLANE), w2 = 3 w1 SPHERE (not LINE)
    t, _, _, cov = typed("one_third", "plane tie")
    w = np.sort(np.diag(cov).astype(np.float64))
    assert np.count_nonzero(cov - np.diag(np.diag(cov))) == 0 and w[1] * (1.0 / 3.0) == w[0] and t == K_LINE
    t, _, _, cov = typed("one_third", "line tie")
    w = np.sort(np.diag(cov).astype(np.float64))
    assert np.count_nonzero(cov - np.diag(np.diag(cov))) == 0 and w[2] * (1.0 / 3.0) == w[1] and w[1] * (1.0 / 3.0) < w[0] and t == K_SPHERE
    # one float either side of each boundary: the oracle's type flips between the two coordinates
    for rule, want in (("plane", (K_PLANE, K_LINE)), ("line", (K_LINE, K_SPHERE))):
        (ia, pa), (ib, pb) = get[("one_third", f"{rule} flip below")], get[("one_third", f"{rule} flip above")]
        a, b = KC.one_third_flip(KC.centre(*ia), 2 if rule == "plane" else 1), KC.one_third_flip(KC.centre(*ib), 2 if rule == "plane" else 1)
        assert np.array_equal(pa, KC.six_axes(KC.centre(*ia), *a[0])) and np.array_equal(pb, KC.six_axes(KC.centre(*ib), *b[1]))
        assert {typed("one_third", f"{rule} flip below")[0], typed("one_third", f"{rule} flip above")[0]} <= set(want) | {K_SPHERE}
        for e, (lo, hi) in ((ia, a), (ib, b)):
            tl = K.cell_type(KC.six_axes(KC.centre(*e), *lo), KC.centre(*e))[0]
            th = K.cell_type(KC.six_axes(KC.centre(*e), *hi), KC.centre(*e))[0]
            assert tl != th and sum(x != y for x, y in zip(lo, hi)) == 1
    # identical points: the covariance is rounding noise
    assert not typed("identical_points", "5 x 0.3: zero covariance")[3].any()
    cov = typed("identical_points", "7 x 0.7: rank 1, three equal entries")[3]
    assert len(np.unique(cov)) == 1 and cov[0, 0] != 0
    cov = typed("identical_points", "5 x 123.456: a negative eigenvalue")[3]
    assert np.linalg.eigvalsh(cov.astype(np.float64)).min() < 0
    # axis-aligned: the vector is exactly an axis; the diagonal lines pin the first of equal components positive
    for a in range(3):
        for kind, want in (("line", K_LINE), ("plane", K_PLANE)):
            t, v, _, _ = typed("axis_aligned", f"{kind} axis {a}")
            assert t == want and np.array_equal(v, np.eye(3, dtype=np.float32)[a])
    for what, sy in (("line (1, 1, 0)", 1), ("line (1, -1, 0)", -1)):
        t, v, _, _ = typed("axis_aligned", what)
        assert t == K_LINE and v[0] > 0 and v[1] == sy * v[0] and v[2] == 0
    # the centre gate: the mean one float inside 0.375, at it exactly (typed), one float outside (not typed)
    for s, (want_d, want_t) in enumerate(((-1, K_PLANE), (0, K_PLANE), (1, K_SPHERE))):
        ijk, p = get[("centre_gate", ["gate below", "gate at", "gate above"][s])]
        c = KC.centre(*ijk)
        _, _, m, _ = K.cell_type(p, c)
        e = (c - m).astype(np.float32)
        dn = np.sqrt(np.float32(e[0] * e[0] + np.float32(e[1] * e[1] + e[2] * e[2])))
        assert np.sign(dn - np.float32(0.375)) == want_d and K.cell_type(p, c)[0] == want_t
    # far cells: how often the float covariance types a cell differently from the exact one (reported, not asserted)
    differ = sum(K.cell_type(p, KC.centre(*ijk))[0] != _fp64_type(p, KC.centre(*ijk).astype(np.float64)) for ijk, p, _ in cc["far_cells"])
    print(f"far cells: {differ} of {len(cc['far_cells'])} typed differently from the fp64 typing")
    assert len(cc["big_cell"][0][1]) >= 100000


@pytest.mark.parametrize("name", list(KC.direction_cases()))
def test_direction_cases_paint_their_designed_images(name):
    cloud, want_line, want_plane = KC.direction_cases()[name]
    m, k = _oracle_keyframe(cloud)
    _, _, typ, vec = m.cells(k)
    imgs, info = m.images(k), m.info(k)
    assert np.array_equal(imgs[0], want_line) and np.array_equal(imgs[1], want_plane)
    cl, cp, frame = K.numpy_images(typ, vec)
    assert np.array_equal(cl, imgs[0]) and np.array_equal(cp, imgs[1])
    assert info["ratio_line"] == np.float32((want_line >= 1).sum()) / np.float32(3600)
    for a in (0, 1):
        assert np.abs(imgs[2 + a] - K.fp64_blur(imgs[a])).max() <= 1e-6 * max(1.0, float(imgs[a].max()))
    if name.startswith("clamps"):
        lines = frame[typ == K_LINE]
        # x' = +0 on every axis line that is not along the image's x' axis; asin(-1) with the identity basis, asin(+1) with +y normals
        assert (np.abs(lines[:, 2]) == 1).sum() == 1 and not np.signbit(lines[:, 0]).any()
        assert lines[np.abs(lines[:, 2]) == 1][0, 2] == (1 if name == "clamps_y_normals" else -1)


def test_growth_appends_reach_their_edges():
    m = K.OracleMap(1.0, revisit_threshold=2)
    ks = [m.new_keyframe(), m.new_keyframe()]
    sizes = []
    for cloud, op in KC.growth_appends():
        m.append(cloud, [ks[i] for i in op])
        sizes.append(m.info(ks[0])["cells"])
    assert sizes[1] <= 4096 < sizes[-1] and m.info(ks[1])["cells"] < sizes[-1]
    keys, inc, _, _ = m.cells(ks[0])
    assert inc.max() == 1 and len(np.unique(keys)) == len(keys) - 1   # the revisited cell held in both incarnations


@pytest.mark.parametrize("name", list(KC.roi_cases()))
def test_roi_cases_equal_numpy(name):
    cloud = KC.roi_cases()[name]
    m, k = _oracle_keyframe(cloud)
    c, roi = K.numpy_roi_range(np.array([KC.centre(*x) for x in sorted(set(map(tuple, KC.cell_of(cloud))), key=lambda x: int(_key(x)))], np.float32))
    info = m.info(k)
    assert np.array_equal(c, info["center"]) and roi == info["roi_range"]


def test_roi_cases_reach_their_edges():
    us = {}
    for name, cloud in KC.roi_cases().items():
        cent = np.array([KC.centre(*x) for x in sorted(set(map(tuple, KC.cell_of(cloud))), key=lambda x: int(_key(x)))], np.float32)
        c = K.numpy_roi_range(cent)[0]
        d = cent - c
        us[name] = len(np.unique(np.sqrt((d[:, 0] * d[:, 0] + (d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])).astype(np.float32))))
        assert len(cent) == (len(cloud) - 1 if name == 'duplicate_distances' else len(cloud))   # one cell taken twice there
    assert us["one_cell"] == 1 and us["cube_corners"] == 1 and us["duplicate_distances"] < 24
    onto = {n: float(np.float32(us[n] - 1) * np.float32(0.9)).is_integer() for n in us if n.startswith("distinct")}
    assert any(onto.values()) and not all(onto.values())


def test_blur_of_a_cyclic_shift_is_the_shifted_blur():
    r = np.random.default_rng(9)
    img = np.zeros((60, 60), np.float32)
    img[0, :] = 1
    img[:, 59] += 2
    img[r.integers(0, 60, 30), r.integers(0, 60, 30)] += 5
    img[17, 42] = 1000
    for s in ((1, 0), (0, 1), (30, 30), (59, 7), (-13, 29)):
        assert np.array_equal(K.blur(np.roll(img, s, (0, 1))), np.roll(K.blur(img), s, (0, 1)))
    assert np.abs(K.blur(img) - K.fp64_blur(img)).max() <= 1e-6 * float(img.max())


@pytest.mark.parametrize("name", ["newest_1", "cyclic_shifts", "zero_and_one_pixel"])
def test_search_cases_oracle_equals_fp64(name):
    kfs = KC.search_cases()[name]
    imgs = []
    for px, planes in kfs:
        cl = np.zeros((60, 60), np.float32)
        for (p, t), n in px.items():
            cl[p, t] = n
        cp = np.zeros((60, 60), np.float32)
        cp[30, 30] = planes
        imgs.append((K.blur(cp), K.blur(cl)))
    a = imgs[-1]
    for b, (px, _) in zip(imgs[:-1], kfs[:-1]):
        for w in (0, 1):
            s = K.similarity(a[w], b[w])
            assert abs(s - K.fp64_similarity(a[w], b[w])) <= 2e-6
    if name == "cyclic_shifts":
        # every cyclic shift of the newest's line image scores exactly 1: the wrap pad reaches every offset, and num = den = sum T^2 bit for bit
        for b, (px, _) in zip(imgs[:-2], kfs[:-2]):
            assert K.similarity(a[1], b[1]) == 1.0
        assert K.similarity(a[1], imgs[-2][1]) < 1.0
