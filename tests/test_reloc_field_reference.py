"""The NumPy restatement of the class-aware distance-field relocalization (tests/reloc_field_reference.py: field, field_scores, fine_group, pick)
against independent formulations, and the ctypes layout of ll_reloc_fine_cfg / ll_reloc_field_candidate against the header (no GPU)."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import scipy.ndimage as ndi
from scipy.spatial.transform import Rotation

import reloc_field_reference as F
import reloc_reference as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _exact_field(occ, T):
    """min(T^2, integer squared distance to the nearest occupied voxel) from scipy's exact EDT and its feature indices."""
    if not occ.any():
        return np.full(occ.shape, T * T, np.uint8)
    _, idx = ndi.distance_transform_edt(~occ, return_indices=True)
    grid = np.indices(occ.shape)
    d2 = ((idx - grid) ** 2).sum(axis=0)
    return np.minimum(d2, T * T).astype(np.uint8)


@pytest.mark.parametrize("T", [1, 2, 5, 15])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_separable_field_is_the_exact_truncated_edt(T, seed):
    rng = np.random.default_rng(100 * T + seed)
    shape = (6 + 3 * seed, 9 + seed, 23 - 4 * seed)
    occ = rng.random(shape) < (0.002, 0.02, 0.2)[seed]
    occ[0, 0, 0] = occ[-1, -1, -1] = True   # voxels on the border
    occ[shape[0] // 2, 0, shape[2] - 1] = True
    assert np.array_equal(F.edt_separable(occ, T), _exact_field(occ, T))


@pytest.mark.parametrize("T", [1, 5, 15])
def test_empty_and_single_voxel_fields(T):
    occ = np.zeros((5, 7, 40), bool)
    assert (F.edt_separable(occ, T) == T * T).all() and (_exact_field(occ, T) == T * T).all()
    occ[2, 3, 0] = True   # one voxel on the x border: the field is the truncated squared distance to it
    z, y, x = np.indices(occ.shape)
    want = np.minimum((z - 2) ** 2 + (y - 3) ** 2 + x ** 2, T * T)
    assert np.array_equal(F.edt_separable(occ, T), want.astype(np.uint8))


def test_field_of_clouds_has_one_anchor_and_an_empty_class():
    rng = np.random.default_rng(7)
    corner = rng.uniform(-3, 1, (50, 4)).astype(np.float32)
    surf = rng.uniform(-1, 4, (80, 4)).astype(np.float32)
    surf[3, :3] = np.nan
    dims, lo, d2 = F.field([corner, surf], 0.5, 3)
    both = np.concatenate([corner, surf])[:, :3]
    both = both[np.all(np.isfinite(both), axis=1)]
    assert np.array_equal(lo, both.min(axis=0)) and dims.tolist() == R.dims_of(lo, both.max(axis=0), 0.5, 3).tolist()
    for cls, cloud in enumerate((corner, surf)):
        c, ok = R.cells(cloud[np.all(np.isfinite(cloud[:, :3]), axis=1)], lo, 0.5, 3, dims)
        assert ok.all() and (d2[cls][c[:, 2], c[:, 1], c[:, 0]] == 0).all()
    dims1, _, d21 = F.field([corner, np.zeros((0, 4), np.float32)], 0.5, 3)
    assert (d21[1] == 9).all() and (d21[0] == 0).sum() > 0


def _field_case(seed, T):
    rng = np.random.default_rng(seed)
    clouds = [rng.uniform(-3, 3, (120, 4)).astype(np.float32), rng.uniform(-2, 4, (300, 4)).astype(np.float32)]
    dims, lo, d2 = F.field(clouds, 0.5, T)
    pts = [rng.uniform(-2, 2, (25, 4)).astype(np.float32), rng.uniform(-2, 2, (30, 4)).astype(np.float32)]
    pts[0][3, :3] = np.nan
    pts[1][4, 0] = np.inf
    pts[1][5, :3] = 0.0
    return dims, lo, d2, pts


@pytest.mark.parametrize("T", [1, 5])
def test_field_scores_equal_a_plain_loop_for_coarse_fine_and_verify_groups(T):
    dims, lo, d2, pts = _field_case(3 + T, T)
    yaw = np.radians([0.0, 40.0, 200.0])
    rot = np.stack([np.cos(yaw / 2), 0 * yaw, 0 * yaw, np.sin(yaw / 2)], axis=1)
    groups = [(rot, (-4.0, -1.0, 0.0), (1.5, 0.7, 0.3), (6, 3, 2))]                                # coarse
    a = np.radians([-3.0, 0.0, 3.0]) * 0.5
    dq = np.stack([np.cos(a), 0 * a, 0 * a, np.sin(a)], axis=1)
    for q, t in ((rot[1], (0.5, -0.25, 0.1)), (rot[2], (-1.0, 1.0, 0.0))):                        # two fine groups
        rf, o = F.fine_group(q, t, dq, (0.1, 0.1, 0.1), (5, 3, 1))
        groups.append((rf, o, (0.1, 0.1, 0.1), (5, 3, 1)))
    qv = np.array([0.9, 0.05, -0.03, 0.4]); qv /= np.linalg.norm(qv)
    groups.append((qv[None], (0.31, -0.77, 0.05), (0.0, 0.0, 0.0), (1, 1, 1)))                  # verify: one pose
    for rr, t0, step, nt in groups:
        x = F.field_scores(d2, dims, lo, 0.5, T, pts, rr, t0, step, nt)
        y = F.field_scores_loop(d2, dims, lo, 0.5, T, pts, rr, t0, step, nt)
        assert x.dtype == np.int32 and np.array_equal(x, y) and x.max() > 0


@pytest.mark.parametrize("chunk", [1, 3, None])
def test_vectorised_field_scores_equal_the_per_hypothesis_scores_and_the_loop(chunk):
    from test_reloc_reference import vec_case
    cloud, pts, rot = vec_case(23)
    surf = np.concatenate([cloud[200:], np.float32([[0.25, 0.5, -0.75, 0]])])
    dims, lo, d2 = F.field([cloud[:200], surf], 0.5, 3)
    sp = [pts[:30], pts[30:]]
    sp[1][0, :3] = (0.25, 0.5, -0.75)   # on the surface class's own voxel face
    for t0, step, nt in (((-1.0, -0.5, 0.0), (0.5, 0.5, 0.5), (5, 3, 2)), ((0.3, 0.2, -0.1), (0.0, 0.0, 0.0), (3, 2, 2)),
                         ((2.0, 1.0, 0.5), (-0.35, -0.5, -0.25), (7, 4, 3))):
        a = F.field_scores_vec(d2, dims, lo, 0.5, 3, sp, rot, t0, step, nt, chunk=chunk)
        b = F.field_scores(d2, dims, lo, 0.5, 3, sp, rot, t0, step, nt)
        assert a.dtype == np.int32 and np.array_equal(a, b) and a.max() > 0
        if chunk == 1:
            assert np.array_equal(a, F.field_scores_loop(d2, dims, lo, 0.5, 3, sp, rot, t0, step, nt))
    # a class without points next to one with points, and no finite point at all
    none = np.zeros((0, 4), np.float32)
    for p in ([none, sp[1]], [sp[0], none], [none, none], [pts[12:15], pts[12:15]]):
        assert np.array_equal(F.field_scores_vec(d2, dims, lo, 0.5, 3, p, rot, (0, 0, 0), (0.5, 0.5, 0.5), (3, 2, 1)),
                              F.field_scores(d2, dims, lo, 0.5, 3, p, rot, (0, 0, 0), (0.5, 0.5, 0.5), (3, 2, 1)))


def test_one_call_pipeline_is_coarse_peaks_fine_groups_and_picks():
    from test_reloc_reference import vec_case
    cloud, pts, rot = vec_case(29)
    dims, lo, d2 = F.field([cloud[:40], cloud[40:100]], 0.5, 1)
    sp = [pts[:20], pts[20:]]
    t0, step, nt = (-2.5, -2.0, 0.0), (0.6, 0.6, 0.5), (9, 9, 1)
    a = np.radians([-4.0, 0.0, 4.0]) * 0.5
    dq = np.stack([np.cos(a), 0 * a, 0 * a, np.sin(a)], axis=1)
    fstep, fnt = (0.1, 0.2, 0.1), (5, 3, 1)
    out = F.relocalize_field(d2, dims, lo, 0.5, 1, sp, rot, t0, step, nt, 5, dq, fstep, fnt)
    sc = F.field_scores(d2, dims, lo, 0.5, 1, sp, rot, t0, step, nt)
    hs, ss = R.peaks_brute(sc, 3, nt, True)
    assert np.array_equal(out["scores"], sc) and out["n_peaks"] == hs.shape[0] > 5 and len(out["candidates"]) == 5
    for j, c in enumerate(out["candidates"]):
        assert (c["hypothesis"], c["score"]) == (hs[j], ss[j])
        q, t = R.candidate_pose(hs[j], rot, t0, step, nt)
        rf, o = F.fine_group(q, t, dq, fstep, fnt)
        fs = F.field_scores(d2, dims, lo, 0.5, 1, sp, rf, o, fstep, fnt)
        i = max(range(fs.shape[0]), key=lambda k: (fs[k], -k))
        fq, ft = F.fine_pose(rf, o, fstep, fnt, i)
        assert np.array_equal(out["fine"][j], fs) and (c["fine_index"], c["fine_score"]) == (i, fs[i])
        assert np.array_equal(c["q"], q) and np.array_equal(c["t"], t) and np.array_equal(c["fine_q"], fq) and np.array_equal(c["fine_t"], ft)
    v = F.verify_scores(d2, dims, lo, 0.5, 1, sp, [(c["fine_q"], c["fine_t"]) for c in out["candidates"]])
    assert v == [c["fine_score"] for c in out["candidates"]]   # the verify score of a fine pose is its fine score


def test_field_score_is_class_aware():
    T = 3
    corner = np.array([[0.0, 0.0, 0.0, 0]], np.float32)
    surf = np.array([[4.0, 0.0, 0.0, 0]], np.float32)
    dims, lo, d2 = F.field([corner, surf], 0.5, T)
    at_c, at_s = np.array([[0.1, 0.1, 0.1, 0]], np.float32), np.array([[4.1, 0.1, 0.1, 0]], np.float32)
    one = np.array([[1.0, 0, 0, 0]])
    sc = lambda c, s: int(F.field_scores(d2, dims, lo, 0.5, T, [c, s], one, (0, 0, 0), (1, 1, 1), (1, 1, 1))[0])   # noqa: E731
    none = np.zeros((0, 4), np.float32)
    assert sc(at_c, none) == 9 and sc(none, at_s) == 9          # each class on its own structure: T^2
    assert sc(at_s, none) == 0 and sc(none, at_c) == 0          # on the other class's structure: nothing
    half = np.array([[0.6, 0.1, 0.1, 0]], np.float32)           # one voxel away: T^2 - 1
    assert sc(half, none) == 8


def test_fine_group_is_the_stated_host_formula():
    rng = np.random.default_rng(11)
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    dq = rng.normal(size=(5, 4)); dq /= np.linalg.norm(dq, axis=1, keepdims=True)
    t, step, nt = (10.25, -0.47, 0.1), (0.1, 0.2, 0.3), (11, 5, 1)
    rot, o = F.fine_group(q, t, dq, step, nt)
    for r in range(5):
        w1, x1, y1, z1 = q
        w2, x2, y2, z2 = dq[r]
        want = [w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2, w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2]
        assert rot[r].tolist() == want
        # q (x) dq is the rotation dq applied first, then q
        m = (Rotation.from_quat(np.roll(q, -1)) * Rotation.from_quat(np.roll(dq[r], -1))).as_quat()
        assert min(np.abs(np.roll(rot[r], -1) - m).max(), np.abs(np.roll(rot[r], -1) + m).max()) < 1e-12
    assert o.tolist() == [10.25 - 5.0 * 0.1, -0.47 - 2.0 * 0.2, 0.1 - 0.0 * 0.3]
    qf, tf = F.fine_pose(rot, o, step, nt, 5 + 11 * (2 + 5 * 0) + 55 * 3)
    assert np.array_equal(qf, rot[3]) and tf.tolist() == [o[0] + 5.0 * 0.1, o[1] + 2.0 * 0.2, o[2]]
    assert F.pick([3, 7, 2, 7, 7]) == (1, 7) and F.pick([0, 0]) == (0, 0)


def test_fine_search_defaults():
    from loam_livox_b200.registration import fine_search
    dq, step, nt = fine_search(10.0, ((-1.0, 39.0, 1.0), (-5.0, 5.0, 1.0), (0.1, 0.1, 0.0)))
    yaw = np.degrees(2 * np.arctan2(dq[:, 3], dq[:, 0]))
    assert dq.shape == (11, 4) and np.allclose(yaw, np.arange(-5, 6)) and np.allclose(np.linalg.norm(dq, axis=1), 1.0)
    assert step == [0.1, 0.1, 0.1] and nt == [31, 31, 1]
    assert fine_search(10.0, ((-1.0, 39.0, 1.0), (-5.0, 5.0, 1.0), (0.1, 0.1, 0.0)), fine_t_half=0.5)[2] == [11, 11, 1]
    dq2, _, nt2 = fine_search(30.0, ((0.0, 2.0, 0.5), (0.0, 0.0, 0.0), (0.0, 1.0, 0.3)), fine_yaw_step_deg=2.0, fine_t_step=0.1, fine_t_half=0.5)
    assert dq2.shape == (15, 4) and nt2 == [5, 1, 3]


def _header_struct(name):
    txt = open(os.path.join(ROOT, "include", "loamlivox_b200.h")).read()
    m = re.search(r"typedef struct \{([^{}]*)\} " + name + ";", txt)
    assert m, name
    body = re.sub(r"/\*.*?\*/", "", m.group(1), flags=re.S)
    return " ".join(ln.strip() for ln in body.split(";") if ln.strip())


def test_ctypes_layout_matches_header():
    from loam_livox_b200 import capi
    for cls, name, size in ((capi.RelocFineCfg, "ll_reloc_fine_cfg", 56), (capi.RelocFieldCandidate, "ll_reloc_field_candidate", 136)):
        decl = _header_struct(name)
        names = [f for f, _ in cls._fields_]
        pos = [re.search(r"[\s*]" + n + r"\b", " " + decl).start() for n in names]
        assert pos == sorted(pos), name
        assert C.sizeof(cls) == size, name
    assert [f for f, _ in capi.RelocFineCfg._fields_] == ["n_rot", "rot_wxyz", "step", "nt"]
    assert capi.RelocFineCfg.step.offset == 16 and capi.RelocFineCfg.nt.offset == 40
    assert capi.RelocFieldCandidate.fine_q_wxyz.offset == 64 and capi.RelocFieldCandidate.fine_score.offset == 120
    assert capi.RelocFieldCandidate.verify_score.offset == 128
