"""Host-only checks of loop feedback (ll_mapper_set_loop_feedback, ll_mapper_loop_correction_read, ll_loop_correction; DESIGN.md §4.6.2): the
correction rule against its restatement (tests/loop_feedback_reference.py) and scipy's slerp at every edge of the rule; version-3 loop images
through ll_loop_image_info, every rule of their FEEDBACK section just inside and just outside its bound, versions 1 and 2 unchanged; the C ABI,
its ctypes and Python mirrors and the C++ mirror."""
import ctypes as C
import struct
import subprocess

import numpy as np
import pytest
from scipy.spatial.transform import Rotation, Slerp

import loop_feedback_reference as R
from loam_livox_b200 import capi
from loam_livox_b200.registration import loop_correction
from test_loop_image import image, pose, scalars, summary
from test_loop_policy import loop2, parts_k, v2
from test_recovery_cabi import _compile, _header_params


def _random_poses(rng, n, angle=0.4):
    q = Rotation.from_rotvec(rng.normal(size=(n, 3)) * angle).as_quat()[:, [3, 0, 1, 2]]
    return np.concatenate([q, rng.normal(size=(n, 3)) * 3], axis=1)


def _lib(ori, opt, f, s):
    return loop_correction(ori, opt, f, s)


def _ref(ori, opt, f, s):
    q, t = R.correction(ori, opt, list(f), s)
    return np.array(q), np.array(t)


def _scipy(ori, opt, f, s):
    """an independent statement: A_k from rotation matrices, scipy's Slerp between the neighbours, the translations interpolated linearly"""
    def A(k):
        if k == 0:
            return Rotation.identity(), np.zeros(3)
        ro, rp = Rotation.from_quat(ori[k, [1, 2, 3, 0]]), Rotation.from_quat(opt[k, [1, 2, 3, 0]])
        r = rp * ro.inv()
        return r, opt[k, 4:] - r.apply(ori[k, 4:])
    n = len(f)
    if s <= f[0]:
        return A(0)
    if s >= f[-1]:
        return A(n - 1)
    k = max(j for j in range(n) if f[j] <= s)
    (ra, ta), (rb, tb) = A(k), A(k + 1)
    u = (s - f[k]) / (f[k + 1] - f[k])
    return Slerp([0.0, 1.0], Rotation.concatenate([ra, rb]))([u])[0], ta + u * (tb - ta)


def _close(lib, sc):
    (q, t), (r, tt) = lib, sc
    return Rotation.from_quat(q[[1, 2, 3, 0]]).inv() * r, np.abs(t - tt).max()


# ---------------------------------------------------------------------------------------------- the rule
@pytest.mark.parametrize("n", [2, 3, 7])
def test_rule_equals_its_restatement_and_scipy_at_every_edge(n):
    rng = np.random.default_rng(40 + n)
    ori, opt = _random_poses(rng, n), _random_poses(rng, n)
    opt[0] = ori[0]
    f = np.cumsum(rng.integers(1, 9, n)) + 3
    steps = sorted({0, int(f[0]) - 1, int(f[-1]) + 1, int(f[-1]) + 40} | {int(x) + d for x in f for d in (-1, 0, 1)} | {int((f[0] + f[-1]) // 2)})
    for s in steps:
        q, t = _lib(ori, opt, f, s)
        rq, rt = _ref(ori, opt, f, s)
        assert q.tobytes() == rq.tobytes() and t.tobytes() == rt.tobytes(), s
        dr, dt = _close((q, t), _scipy(ori, opt, f, s))
        assert dr.magnitude() < 1e-9 and dt < 1e-9, (s, dr.magnitude(), dt)
        if s <= f[0]:
            assert q.tolist() == [1, 0, 0, 0] and t.tolist() == [0, 0, 0]
    # at f[k] exactly: A_k, whatever lies around it
    for k in range(1, n):
        q, t = _lib(ori, opt, f, int(f[k]))
        a = R.keyframe_correction(ori, opt, k)
        assert q.tolist() == list(a[0]) and t.tolist() == list(a[1])


def test_rotations_near_half_a_turn_and_the_sign_of_q():
    rng = np.random.default_rng(9)
    ori = np.zeros((3, 7)); ori[:, 0] = 1; ori[:, 4:] = rng.normal(size=(3, 3))
    opt = ori.copy()
    # A_1 and A_2 turn by 179.9 and 180 degrees about nearby axes; A_2 stored as -q, so the shorter arc needs the sign flipped
    for k, deg, axis in ((1, 179.9, [0, 0, 1]), (2, 180.0, [0.05, 0, 1])):
        qa = Rotation.from_rotvec(np.radians(deg) * np.array(axis) / np.linalg.norm(axis)).as_quat()[[3, 0, 1, 2]]
        opt[k, :4] = qa if k == 1 else -qa
    f = [2, 10, 20]
    for s in (11, 15, 19):
        q, t = _lib(ori, opt, f, s)
        rq, rt = _ref(ori, opt, f, s)
        assert q.tobytes() == rq.tobytes() and t.tobytes() == rt.tobytes()
        dr, dt = _close((q, t), _scipy(ori, opt, f, s))
        assert dr.magnitude() < 1e-9 and dt < 1e-9, (s, dr.magnitude())
    # -q and q are the same correction
    opt2 = opt.copy(); opt2[2, :4] *= -1
    for s in (11, 15, 19):
        a, b = _lib(ori, opt, f, s), _lib(ori, opt2, f, s)
        assert (Rotation.from_quat(a[0][[1, 2, 3, 0]]).inv() * Rotation.from_quat(b[0][[1, 2, 3, 0]])).magnitude() < 1e-12
        assert np.abs(a[1] - b[1]).max() < 1e-12


def test_an_identity_graph_gives_the_identity():
    rng = np.random.default_rng(3)
    ori = _random_poses(rng, 4)
    f = [5, 9, 14, 30]
    for s in (0, 5, 7, 9, 20, 30, 99):
        q, t = _lib(ori, ori, f, s)
        assert np.abs(q - [1, 0, 0, 0]).max() < 1e-15 and np.abs(t).max() < 1e-14, s


def test_rule_refusals():
    ori = np.tile([1.0, 0, 0, 0, 0, 0, 0], (3, 1))
    L = capi.lib()
    q, t = np.zeros(4), np.zeros(3)
    P = C.POINTER(capi.Pose)
    for f in ([1, 1, 2], [3, 2, 4]):
        fa = np.array(f, np.int32)
        assert L.ll_loop_correction(ori.ctypes.data_as(P), ori.ctypes.data_as(P), fa.ctypes.data, 3, 2, q.ctypes.data, t.ctypes.data) == capi.LL_ERR_INVALID
    fa = np.array([1, 2, 3], np.int32)
    assert L.ll_loop_correction(ori.ctypes.data_as(P), ori.ctypes.data_as(P), fa.ctypes.data, 0, 2, q.ctypes.data, t.ctypes.data) == capi.LL_ERR_INVALID
    assert L.ll_loop_correction(None, ori.ctypes.data_as(P), fa.ctypes.data, 3, 2, q.ctypes.data, t.ctypes.data) == capi.LL_ERR_INVALID
    assert L.ll_loop_correction(ori.ctypes.data_as(P), ori.ctypes.data_as(P), fa.ctypes.data, 3, 2, None, t.ctypes.data) == capi.LL_ERR_INVALID
    with pytest.raises(Exception):
        loop_correction(ori, ori, [1, 1, 2], 2)


def test_the_window_transform_restatement_is_the_transform_kernels_arithmetic():
    """the restated window transform of one point against the same fp64 steps written out by hand"""
    rng = np.random.default_rng(5)
    pts = rng.uniform(-30, 30, (64, 4)).astype(np.float32)
    d = R.pose(_random_poses(rng, 1)[0])
    out = R.transform(pts, d)
    for p, o in zip(pts, out):
        r = R.qrot(d[0], tuple(float(x) for x in p[:3]))
        assert [np.float32(r[k] + d[1][k]) for k in range(3)] + [p[3]] == list(o)


# ---------------------------------------------------------------------------------------------- version-3 loop images
K = 6


def fb_section(on=1, n_applied=2, corr=None, nk=K, f=None, frames=(3, 5, 6, 9), ns=None):
    corr = (0.9, 0.1, 0.3, 0.3, 0.2, -0.1, 0.05) if corr is None else corr
    f = tuple(2 * k + 1 for k in range(K)) if f is None else f
    ns = len(frames) if ns is None else ns
    return struct.pack("<ii7dqq", on, n_applied, *corr, nk, ns) + np.asarray(f, "<i4").tobytes() + np.asarray(frames, "<i4").tobytes()


def v3(fb=None, max_loops=3, gap=2, loops=((2, 0), (4, 1)), stopped=0, frame_index=12, history=400, **kw):
    p = parts_k(K)
    p[11] = loop2(max_loops=max_loops, gap=gap, loops=loops)
    p[1] = scalars(closed=int(len(loops) > 0), n_keyframes=K, stopped=stopped, frame_index=frame_index, history=history)
    p.append(fb_section(**kw) if fb is None else fb)
    return image(p, version=capi.LL_LOOP_IMAGE_VERSION_FEEDBACK)


IDENT = (1.0, 0, 0, 0, 0, 0, 0)


def status(img):
    return summary(img)[0]


def test_valid_version_3_images_are_accepted_and_reported():
    st, got = summary(v3())
    assert st == capi.LL_OK and (got.version, got.closed, got.keyframes) == (3, 1, 6)
    from loam_livox_b200.registration import loop_image_info
    assert loop_image_info(v3())["version"] == 3
    ok = {
        "the default policy": v3(max_loops=1, loops=((2, 0),), n_applied=1),
        "no loop yet, the identity": v3(loops=(), n_applied=0, corr=IDENT),
        "one correction short when stopped": v3(stopped=1, n_applied=1),
        "no window segment": v3(frames=()),
        "frame indices at 0 and at frame_index": v3(f=(0, 1, 2, 3, 4, 12), frames=(0, 12)),
        "segments at maximum_history_size": v3(history=4),
    }
    for name, img in ok.items():
        assert status(img) == capi.LL_OK, name


def test_version_3_refusals():
    bad = {
        "flag 0": v3(on=0),
        "flag 2": v3(on=2),
        "n_applied above n_loops": v3(n_applied=3),
        "negative n_applied": v3(n_applied=-1),
        "one correction short without stopped": v3(n_applied=1),
        "no correction but C not the identity": v3(loops=(), n_applied=0),
        "non-finite C": v3(corr=(1.0, 0, 0, 0, float("nan"), 0, 0)),
        "keyframes other than n_keyframes": v3(nk=K - 1, f=tuple(range(1, K))),
        "keyframe index repeated": v3(f=(1, 3, 3, 7, 9, 11)),
        "keyframe index decreasing": v3(f=(1, 5, 3, 7, 9, 11)),
        "keyframe index negative": v3(f=(-1, 3, 5, 7, 9, 11)),
        "keyframe index past frame_index": v3(f=(1, 3, 5, 7, 9, 13)),
        "segment index repeated": v3(frames=(3, 5, 5, 9)),
        "segment index decreasing": v3(frames=(3, 6, 5, 9)),
        "segment index negative": v3(frames=(-1, 5)),
        "segment index past frame_index": v3(frames=(3, 13)),
        "segments above maximum_history_size": v3(history=3),
        "segment count too large": v3(ns=5),
        "segment count negative": v3(ns=-1),
        "trailing bytes": v3(fb=fb_section() + b"\0" * 4),
        "shorter than its head": v3(fb=fb_section()[:70]),
        "max_loops 0": v3(max_loops=0, loops=(), n_applied=0, corr=IDENT),
    }
    for name, img in bad.items():
        assert status(img) == capi.LL_ERR_INVALID, name
    # a version-3 header without its fourteenth section
    p = parts_k(K)
    p[11] = loop2()
    p[1] = scalars(closed=1, n_keyframes=K)
    assert status(image(p, version=3)) == capi.LL_ERR_INVALID


def test_versions_1_and_2_are_unchanged():
    assert status(v2()) == capi.LL_OK and summary(v2())[1].version == 2
    p = parts_k(K)
    p[1] = scalars(closed=0, n_keyframes=K)
    assert status(image(p)) == capi.LL_OK and summary(image(p))[1].version == 1
    # the header of a version-1 or 2 image is still 24 + 16 * 13 bytes: its first section starts there
    assert struct.unpack_from("<Q", v2(), 24)[0] == 24 + 16 * capi.LL_LOOP_IMAGE_SECTIONS
    assert struct.unpack_from("<Q", v3(), 24)[0] == 24 + 16 * capi.LL_LOOP_IMAGE_SECTIONS_FEEDBACK


def test_the_reader_of_the_feedback_section():
    na, c, f, fr = R.feedback_section(v3())
    assert na == 2 and c[0] == (0.9, 0.1, 0.3, 0.3) and f.tolist() == [1, 3, 5, 7, 9, 11] and fr.tolist() == [3, 5, 6, 9]


# ---------------------------------------------------------------------------------------------- ABI
def test_symbols_signatures_and_refusals_without_a_mapper():
    L = capi.lib()
    for name, n_params in (("ll_mapper_set_loop_feedback", 2), ("ll_mapper_loop_correction_read", 4), ("ll_loop_correction", 7)):
        assert hasattr(L, name) and name in capi.EXPORTS
        assert len(_header_params(name)) == len(getattr(L, name).argtypes) == n_params, name
    q, t, n = np.zeros(4), np.zeros(3), C.c_int()
    assert L.ll_mapper_set_loop_feedback(None, 1) == capi.LL_ERR_INVALID
    assert L.ll_mapper_loop_correction_read(None, q.ctypes.data, t.ctypes.data, C.byref(n)) == capi.LL_ERR_INVALID


def test_constants_equal_the_cpp_header(tmp_path):
    exe = _compile(tmp_path, "loop_feedback_mirror")
    r = subprocess.run([exe, "layout"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    seen = set()
    for line in r.stdout.splitlines():
        kind, name, value = line.split()
        if kind == "const":
            assert getattr(capi, name) == int(value), name
            seen.add(name)
        else:
            assert C.sizeof(capi.Pose) == int(value) == 56
    assert seen == {"LL_LOOP_IMAGE_VERSION_FEEDBACK", "LL_LOOP_IMAGE_FEEDBACK", "LL_LOOP_IMAGE_SECTIONS_FEEDBACK", "LL_LOOP_FEEDBACK_MAX_SEGMENTS",
                    "LL_LOOP_IMAGE_SECTIONS"}


def test_cpp_mirror_loop_feedback_compiles_links_and_runs(tmp_path):
    exe = _compile(tmp_path, "loop_feedback_mirror")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)


@pytest.mark.parametrize("name", ["set_loop_feedback", "loop_correction"])
def test_python_mirrors_exist(name):
    from loam_livox_b200.registration import Laser_mapping
    assert callable(getattr(Laser_mapping, name))
