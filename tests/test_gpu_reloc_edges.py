"""The relocalization kernels (csrc/reloc.cu) against their exact NumPy restatement (tests/reloc_reference.py, tests/reloc_field_reference.py) at the
shipped search sizes and at their tile, group and tie edges, integer for integer and bit for bit: the score kernels across several 1 024-point
tiles and CTAs of 64 translations, the peak kernel on plateaus and short rotation axes, the selection past its first 1 024 peaks, the fine picks
of groups larger than one 1 024-thread pass, and the inputs the streaming mapper's recovery hands to ll_relocalize_field (DESIGN.md §4.3.2).
Every case first asserts the property that makes it an edge case."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from loam_livox_b200 import synthetic as S  # noqa: E402
import reloc_field_reference as F  # noqa: E402
import reloc_reference as R  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "golden_small.npz")
TILE = 1024        # score points per pass of the score kernels (RELOC_TILE)
GROUP = 64         # translations per CTA of the score kernels (RELOC_GROUP)
MAX_PTS = 8192     # LL_RELOC_MAX_SCORE_POINTS
RES, DIL, TR = 0.3, 1, 3
ROOM = ((-1.0, 39.0, 1.0), (-5.0, 5.0, 1.0))


@pytest.fixture(scope="module")
def ctxs():
    from loam_livox_b200.registration import Context
    cs = [Context(0, max_scan_points=200000, max_features=400000) for _ in range(2)]
    yield cs
    for c in cs:
        c.close()


@pytest.fixture(scope="module")
def golden(ctxs):
    """The golden_small map with its occupancy index (0.3 m, dilate 1) and distance fields (0.3 m, T = 3 and T = 1), on the GPU and in NumPy."""
    from loam_livox_b200.registration import Map, RelocField, RelocIndex
    g = np.load(GOLDEN)
    mc, ms = g["map_corner"], g["map_surf"]
    m = Map(ctxs[0], mc, ms)
    out = {"g": g, "map": m, "index": RelocIndex(ctxs[0], m, RES, DIL, 1 << 17), "field": RelocField(ctxs[0], m, RES, TR, 1 << 17),
           "field1": RelocField(ctxs[0], m, RES, 1, 1 << 17), "occ": R.index([mc, ms], RES, DIL)[:3], "d2": F.field([mc, ms], RES, TR),
           "d2_1": F.field([mc, ms], RES, 1)}
    yield out
    for k in ("index", "field", "field1"):
        out[k].close()


def _near_map(g, n, seed, which=None):
    """n float32 score points drawn (with repetition) from the map's points, 5 cm of noise added: they score near the identity pose."""
    src = np.concatenate([g["map_corner"], g["map_surf"]]) if which is None else g[which]
    rng = np.random.default_rng(seed)
    p = src[rng.integers(0, src.shape[0], n)].copy()
    p[:, :3] += rng.normal(0.0, 0.05, (n, 3)).astype(np.float32)
    return np.ascontiguousarray(p, np.float32)


def _poison(p, idx=(TILE - 1, TILE, MAX_PTS - 1)):
    """NaN / inf coordinates at the tile boundaries that lie inside p."""
    bad = ((np.nan, 0.0, 0.0), (0.0, np.inf, 0.0), (0.0, 0.0, -np.inf))
    for i, b in zip(idx, bad):
        if i < p.shape[0]:
            p[i, :3] = b
    return p


def _yaws(deg):
    a = np.radians(np.asarray(deg, np.float64)) * 0.5
    return np.stack([np.cos(a), 0 * a, 0 * a, np.sin(a)], axis=1)


def _rot3():
    tilt = S.quat_from_euler(0.03, -0.02, 0.0)
    return np.array([[1.0, 0.0, 0.0, 0.0], S.quat_mul(_yaws([2.0])[0], tilt), [0.0, 0.0, 0.0, 1.0]])   # (the last: 180 deg yaw, w = 0 exactly)


def _occ_scores(ctx, G, pts, rot, t0, step, nt):
    from loam_livox_b200.registration import reloc_scores
    got = reloc_scores(ctx, G["index"], pts, rot, t0, step, nt)
    d, lo, grid = G["occ"]
    return got, R.scores_vec(grid, d, lo, RES, DIL, pts, rot, t0, step, nt)


def _field_scores(ctx, G, pts, rot, t0, step, nt, key="field"):
    from loam_livox_b200.registration import reloc_field_scores
    got = reloc_field_scores(ctx, G[key], pts[0], pts[1], rot, t0, step, nt)
    dims, lo, d2 = G["d2" if key == "field" else "d2_1"]
    return got, F.field_scores_vec(d2, dims, lo, RES, TR if key == "field" else 1, pts, rot, t0, step, nt)


SMALL = ((-0.2, -0.1, -0.05), (0.1, 0.1, 0.05), (3, 2, 2))


# ---------------------------------------------------------------------------------------------- the score kernels: tiles
@pytest.mark.parametrize("n", [0, 1, TILE - 1, TILE, TILE + 1, 2 * TILE + 1, MAX_PTS])
def test_occupancy_scores_across_tiles(ctxs, golden, n):
    from loam_livox_b200 import capi
    assert capi.LL_RELOC_MAX_SCORE_POINTS == MAX_PTS
    pts = _poison(_near_map(golden["g"], n, seed=n))
    rot = _rot3()[:2]
    got, want = _occ_scores(ctxs[0], golden, pts, rot, *SMALL)
    assert got.dtype == np.int32 and np.array_equal(got, want)
    if n > 0:
        assert want.max() > 0
    if n > TILE:   # the sum over tiles matters: neither the first tile alone nor the last one alone gives it
        d, lo, grid = golden["occ"]
        last = (n - 1) // TILE * TILE
        for part in (pts[:TILE], pts[last:]) if n > TILE + 1 else (pts[last:],):   # (point 1 024 of 1 025 is inf)
            assert not np.array_equal(R.scores_vec(grid, d, lo, RES, DIL, part, rot, *SMALL), want)


@pytest.mark.parametrize("n_sc,n_ss", [(0, MAX_PTS), (TILE + 1, 1), (MAX_PTS, MAX_PTS), (1, 0), (TILE, TILE - 1), (2 * TILE + 1, 0), (0, 0)])
def test_field_scores_across_tiles_and_classes(ctxs, golden, n_sc, n_ss):
    pts = (_poison(_near_map(golden["g"], n_sc, 7 + n_sc, "map_corner")), _poison(_near_map(golden["g"], n_ss, 11 + n_ss, "map_surf")))
    rot = _rot3()[:2]
    got, want = _field_scores(ctxs[0], golden, pts, rot, *SMALL)
    assert got.dtype == np.int32 and np.array_equal(got, want)
    dims, lo, d2 = golden["d2"]
    tiles = [(c, b) for c, p in enumerate(pts) for b in range(0, p.shape[0], TILE)]
    if len(tiles) > 1:   # the sum over tiles and classes matters: no single tile gives it
        for c, b in (tiles[0], tiles[-1]):
            part = [p[b:b + TILE] if k == c else p[:0] for k, p in enumerate(pts)]
            assert not np.array_equal(F.field_scores_vec(d2, dims, lo, RES, TR, part, rot, *SMALL), want)
    assert want.any() == (n_sc + n_ss > 0)


# ---------------------------------------------------------------------------------------------- the score kernels: lattices and rotations
def _nts():
    out = [(1, 1, 1)]
    for a, b in ((7, 9), (8, 8), (5, 13), (3, 43)):   # n_lat 63, 64, 65, 129
        out += [(a, b, 1), (a, 1, b), (1, a, b)]
    return out


@pytest.mark.parametrize("nt", _nts())
def test_scores_over_ctas_and_rotations(ctxs, golden, nt):
    n_lat = int(np.prod(nt))
    assert n_lat in (1, 63, 64, 65, 129) and 1 in nt
    pts = _near_map(golden["g"], 300, seed=n_lat)
    rot = _rot3()
    t0, step = (-0.2, -0.3, -0.2), (0.07, 0.05, 0.03)
    got, want = _occ_scores(ctxs[0], golden, pts, rot, t0, step, nt)
    assert np.array_equal(got, want) and want.max() > 0
    got, want = _field_scores(ctxs[0], golden, (pts[:100], pts[100:]), rot, t0, step, nt)
    assert np.array_equal(got, want) and want.max() > 0


def test_step_zero_gives_exact_ties(ctxs, golden):
    pts = _near_map(golden["g"], 500, seed=3)
    rot = _rot3()
    for got, want in (_occ_scores(ctxs[0], golden, pts, rot, (0.1, -0.1, 0.0), (0.0, 0.0, 0.0), (4, 3, 2)),
                      _field_scores(ctxs[0], golden, (pts[:200], pts[200:]), rot, (0.1, -0.1, 0.0), (0.0, 0.0, 0.0), (4, 3, 2))):
        assert np.array_equal(got, want)
        per_rot = want.reshape(3, 24)
        assert (per_rot == per_rot[:, :1]).all() and want.max() > 0   # every translation of a rotation is the same one


@pytest.mark.parametrize("rot_name", ["180", "two", "three", "360"])
def test_rotation_counts(ctxs, golden, rot_name):
    from loam_livox_b200.registration import yaw_circle
    rot = {"180": np.array([[0.0, 0.0, 0.0, 1.0]]), "two": _rot3()[[0, 2]], "three": _yaws([0.0, 120.0, 240.0]), "360": yaw_circle(1.0)}[rot_name]
    pts = _near_map(golden["g"], 200, seed=len(rot))
    t0, step, nt = (-0.1, 0.0, 0.0), (0.2, 0.1, 0.1), (2, 1, 1)
    got, want = _occ_scores(ctxs[0], golden, pts, rot, t0, step, nt)
    assert got.shape[0] == 2 * len(rot) and np.array_equal(got, want) and want.max() > 0
    got, want = _field_scores(ctxs[0], golden, (pts[:50], pts[50:]), rot, t0, step, nt)
    assert np.array_equal(got, want) and want.max() > 0


def test_q_and_minus_q_score_the_same(ctxs, golden):
    from loam_livox_b200.registration import reloc_field_scores, reloc_scores
    rot = np.concatenate([_rot3(), _yaws([37.0, -100.0])])
    pts = _near_map(golden["g"], 1500, seed=5)
    a = reloc_scores(ctxs[0], golden["index"], pts, rot, *SMALL)
    b = reloc_scores(ctxs[0], golden["index"], pts, -rot, *SMALL)
    assert np.array_equal(a, b) and a.max() > 0
    a = reloc_field_scores(ctxs[0], golden["field"], pts[:600], pts[600:], rot, *SMALL)
    b = reloc_field_scores(ctxs[0], golden["field"], pts[:600], pts[600:], -rot, *SMALL)
    assert np.array_equal(a, b) and a.max() > 0


def test_max_hypotheses_is_accepted_and_one_more_is_refused(ctxs, golden):
    from loam_livox_b200.registration import LoamLivoxError, RelocField, RelocIndex, reloc_field_scores, reloc_scores
    idx, fld = RelocIndex(ctxs[0], golden["map"], RES, DIL, 1001), RelocField(ctxs[0], golden["map"], RES, TR, 1001)
    pts = _near_map(golden["g"], 300, seed=9)
    rot = np.concatenate([_rot3(), _yaws([10.0, 20.0, 30.0, 40.0])])   # 7 x 11 x 13 = 1001
    t0, step = (-0.3, -0.3, 0.0), (0.05, 0.05, 0.1)
    d, lo, grid = golden["occ"]
    dims, flo, d2 = golden["d2"]
    assert np.array_equal(reloc_scores(ctxs[0], idx, pts, rot, t0, step, (11, 13, 1)), R.scores_vec(grid, d, lo, RES, DIL, pts, rot, t0, step, (11, 13, 1)))
    fp = (pts[:100], pts[100:])
    assert np.array_equal(reloc_field_scores(ctxs[0], fld, *fp, rot, t0, step, (11, 13, 1)), F.field_scores_vec(d2, dims, flo, RES, TR, fp, rot, t0, step, (11, 13, 1)))
    for r, nt in ((rot[:2], (167, 3, 1)), (rot[:1], (1002, 1, 1))):   # 1 002 hypotheses; 1 002 translations
        with pytest.raises(LoamLivoxError):
            reloc_scores(ctxs[0], idx, pts, r, t0, step, nt)
        with pytest.raises(LoamLivoxError):
            reloc_field_scores(ctxs[0], fld, *fp, r, t0, step, nt)
    idx.close(); fld.close()


# ---------------------------------------------------------------------------------------------- peaks and the selection, through the calls
def _state():
    from loam_livox_b200 import capi
    st = capi.default_reg_state()
    st.current_frame_index = st.mapping_init_accumulate_frames + 1
    return st


def _feats(g):
    return np.ascontiguousarray(g["feat_corner"][:20], np.float32), np.ascontiguousarray(g["feat_surf"][:100], np.float32)


def _call_occ(ctx, G, sp, rot, t0, step, nt, K, cyclic):
    """ll_relocalize: (n_cand, best, [(hypothesis, score, q, t)])."""
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import reloc_cfg
    fc, fs = _feats(G["g"])
    sp = np.ascontiguousarray(sp, np.float32)
    cfg, _keep = reloc_cfg(rot, t0, step, nt, K, cyclic)
    cand, res, status = (capi.RelocCandidate * K)(), (capi.RegResult * K)(), (C.c_int * K)()
    n, best = C.c_int(), C.c_int()
    st = _state()
    ctx.check(ctx._lib.ll_relocalize(ctx.h, G["map"].h, G["index"].h, sp.ctypes.data, sp.shape[0], fc.ctypes.data, fc.shape[0], fs.ctypes.data, fs.shape[0],
                                     capi.LL_FMT_XYZI16, capi.LL_HOST, C.byref(cfg), C.byref(st), cand, res, status, C.byref(n), C.byref(best)))
    return n.value, best.value, [(cand[i].hypothesis, cand[i].score, np.array(cand[i].q_wxyz), np.array(cand[i].t)) for i in range(n.value)]


def _call_field(ctx, G, sp, rot, t0, step, nt, K, cyclic, dq=None, fstep=(0.1, 0.1, 0.1), fnt=(1, 1, 1), key="field", m=None):
    """ll_relocalize_field: (n_cand, best, [candidate dicts], refined, item_status)."""
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import fine_cfg, reloc_cfg
    fc, fs = _feats(G["g"])
    sp = [np.ascontiguousarray(p, np.float32) for p in sp]
    cfg, _k1 = reloc_cfg(rot, t0, step, nt, K, cyclic)
    fcfg, _k2 = fine_cfg(np.array([[1.0, 0, 0, 0]]) if dq is None else dq, fstep, fnt)
    cand, res, status = (capi.RelocFieldCandidate * K)(), (capi.RegResult * K)(), (C.c_int * K)()
    n, best = C.c_int(), C.c_int()
    st = _state()
    ctx.check(ctx._lib.ll_relocalize_field(ctx.h, G["map"].h, G[key].h, sp[0].ctypes.data, sp[0].shape[0], sp[1].ctypes.data, sp[1].shape[0], fc.ctypes.data,
                                           fc.shape[0], fs.ctypes.data, fs.shape[0], capi.LL_FMT_XYZI16, capi.LL_HOST, C.byref(cfg), C.byref(fcfg), C.byref(st),
                                           cand, res, status, C.byref(n), C.byref(best)))
    cands = [{"hypothesis": x.hypothesis, "score": x.score, "q": np.array(x.q_wxyz), "t": np.array(x.t), "fine_index": x.fine_index, "fine_score": x.fine_score,
              "fine_q": np.array(x.fine_q_wxyz), "fine_t": np.array(x.fine_t), "verify_score": x.verify_score} for x in (cand[i] for i in range(n.value))]
    return n.value, best.value, cands, [res[i] for i in range(n.value)], [status[i] for i in range(n.value)]


def _same_candidates(got, want, fine=True):
    keys = ("hypothesis", "score", "fine_index", "fine_score") if fine else ("hypothesis", "score")
    assert [tuple(c[k] for k in keys) for c in got] == [tuple(w[k] for k in keys) for w in want]
    for c, w in zip(got, want):
        for k in (("q", "t", "fine_q", "fine_t") if fine else ("q", "t")):
            assert np.array_equal(c[k], w[k]), k


def _peak_case(G, name):
    """(score points, rotations, t0, step, nt, K, cyclic) of a named selection case."""
    g = G["g"]
    if name == "one point":   # scores of 0 and 1: plateaus
        return _near_map(g, 1, 2), _rot3(), (-0.3, -0.2, 0.0), (0.1, 0.1, 0.1), (7, 5, 1), 16, True
    if name == "step 0":
        return _near_map(g, 300, 3), _rot3(), (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), (3, 3, 1), 8, True
    if name.startswith("n_rot"):
        n_rot, cyc = int(name.split()[1]), name.endswith("cyclic")
        rot = np.array([[1.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0, 1.0], _rot3()[1]])   # rotations 0 and 2 alike: on a circle of 3 they compete
        return _near_map(g, 150, 7), rot[:n_rot], (-0.6, -0.45, 0.0), (0.15, 0.15, 0.1), (9, 7, 1), 16, cyc
    if name == "many peaks":
        return _near_map(g, 60, 1), np.array([[1.0, 0, 0, 0]]), (-20.0, -8.0, -3.0), (0.43, 0.29, 0.41), (96, 56, 14), 16, True
    if name == "fewer than K":
        return _near_map(g, 1, 6), np.array([[1.0, 0, 0, 0]]), (0.0, 0.0, 0.0), (0.05, 0.1, 0.1), (2, 1, 1), 16, False
    raise KeyError(name)


PEAK_CASES = ["one point", "step 0", "many peaks", "fewer than K"] + [f"n_rot {n} {c}" for n in (1, 2, 3) for c in ("cyclic", "open")]


@pytest.mark.parametrize("name", PEAK_CASES)
def test_candidates_are_the_first_peaks(ctxs, golden, name):
    sp, rot, t0, step, nt, K, cyc = _peak_case(golden, name)
    H = len(rot) * int(np.prod(nt))
    # occupancy: ll_relocalize
    d, lo, grid = golden["occ"]
    want = R.relocalize(grid, d, lo, RES, DIL, sp, rot, t0, step, nt, K, cyclic=cyc)
    n, best, got_occ = _call_occ(ctxs[0], golden, sp, rot, t0, step, nt, K, cyc)
    _same_candidates([{"hypothesis": h, "score": s, "q": q, "t": t} for h, s, q, t in got_occ], want["candidates"], fine=False)
    assert n == min(K, want["n_peaks"]) and (best >= 0) == (n > 0)
    n_occ, best_occ, occ_peaks = n, best, want["n_peaks"]
    if H <= 4096:
        hb, sb = R.peaks_brute(want["scores"], len(rot), nt, cyc)
        assert [(c["hypothesis"], c["score"]) for c in want["candidates"]] == list(zip(hb[:K].tolist(), sb[:K].tolist()))
    # distance field (T = 1 for the many-peaks case: a field of T = 3 is too smooth to have more than 1 024 peaks here)
    key = "field1" if name == "many peaks" else "field"
    dims, flo, d2 = golden["d2_1" if key == "field1" else "d2"]
    fp = (sp[:len(sp) // 3], sp[len(sp) // 3:])
    wf = F.relocalize_field(d2, dims, flo, RES, 1 if key == "field1" else TR, fp, rot, t0, step, nt, K, np.array([[1.0, 0, 0, 0]]), (0.1, 0.1, 0.1), (1, 1, 1),
                            cyclic=cyc)
    n, best, got, _, _ = _call_field(ctxs[0], golden, fp, rot, t0, step, nt, K, cyc, key=key)
    _same_candidates(got, wf["candidates"])
    assert n == min(K, wf["n_peaks"])
    if H <= 4096:
        hb, sb = R.peaks_brute(wf["scores"], len(rot), nt, cyc)
        assert [c["hypothesis"] for c in wf["candidates"]] == hb[:K].tolist()
    # the property each case stands for
    if name in ("one point", "step 0"):
        sc = want["scores"]
        assert any(np.count_nonzero(sc == s) > 1 for s in np.unique(sc[sc > 0]))   # plateaus of equal positive scores
    elif name == "many peaks":
        assert occ_peaks > TILE and wf["n_peaks"] > TILE and K == 16
    elif name == "fewer than K":
        assert 0 < occ_peaks < K and 0 < wf["n_peaks"] < K
    elif name.startswith("n_rot 3"):   # the wrap decides: cyclic and open differ on this field
        other = R.peaks(want["scores"], 3, nt, not cyc)[0]
        assert not np.array_equal(R.peaks(want["scores"], 3, nt, cyc)[0], other)
    elif name.startswith("n_rot"):   # wrapping starts at 3 rotations: below that the library gives the same candidates with either flag
        o_occ = _call_occ(ctxs[0], golden, sp, rot, t0, step, nt, K, not cyc)
        assert o_occ[:2] == (n_occ, best_occ) and all(a[:2] == b[:2] and np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3])
                                                     for a, b in zip(o_occ[2], got_occ, strict=True))
        o_f = _call_field(ctxs[0], golden, fp, rot, t0, step, nt, K, not cyc, key=key)
        assert o_f[:2] == (n, best)
        _same_candidates(o_f[2], got)


@pytest.mark.parametrize("why", ["non-finite", "outside the grid"])
def test_no_peak_gives_no_candidate(ctxs, golden, why):
    sp = _near_map(golden["g"], 2 * TILE + 5, 8)
    if why == "non-finite":
        sp[:, 0] = np.nan
        t0 = (0.0, 0.0, 0.0)
    else:
        t0 = (1000.0, 0.0, 0.0)
    rot, step, nt = _rot3(), (0.1, 0.1, 0.1), (3, 3, 1)
    got, want = _occ_scores(ctxs[0], golden, sp, rot, t0, step, nt)
    assert not want.any() and np.array_equal(got, want)
    assert _call_occ(ctxs[0], golden, sp, rot, t0, step, nt, 8, True) == (0, -1, [])
    n, best, cands, _, _ = _call_field(ctxs[0], golden, (sp[:TILE + 1], sp[TILE + 1:]), rot, t0, step, nt, 8, True)
    assert (n, best, cands) == (0, -1, [])


# ---------------------------------------------------------------------------------------------- fine picks
def _fine_case(G, name):
    """(dq, fstep, fnt, K, field max_hypotheses or None)."""
    if name == "large group":   # the shipped 11 x 31 x 31
        return _yaws(np.arange(-5, 6)), (0.1, 0.1, 0.1), (31, 31, 1), 2, None
    if name == "one hypothesis":
        return _yaws([0.0]), (0.1, 0.1, 0.1), (1, 1, 1), 4, None
    if name == "step 0":
        return _yaws([-2.0, 0.0, 2.0]), (0.0, 0.0, 0.0), (3, 3, 3), 4, None
    if name == "repeated rotations":
        return _yaws([1.0, 1.0, 1.0]), (0.05, 0.05, 0.05), (3, 1, 1), 4, None
    if name == "K x H_f = max_hypotheses":
        return _yaws([-2.0, 0.0, 2.0]), (0.1, 0.1, 0.1), (7, 7, 1), 4, 4 * 147
    raise KeyError(name)


@pytest.mark.parametrize("name", ["large group", "one hypothesis", "step 0", "repeated rotations", "K x H_f = max_hypotheses"])
def test_fine_picks(ctxs, golden, name):
    from loam_livox_b200.registration import RelocField
    dq, fstep, fnt, K, mh = _fine_case(golden, name)
    sp = _near_map(golden["g"], 900, 12)
    fp = (sp[:200], sp[200:])
    rot, t0, step, nt = _rot3(), (-4.0, -3.0, -0.5), (1.1, 0.9, 0.5), (8, 7, 3)
    G = dict(golden)
    if mh is not None:
        G["field"] = RelocField(ctxs[0], golden["map"], RES, TR, mh)
        assert K * len(dq) * int(np.prod(fnt)) == mh and len(rot) * int(np.prod(nt)) <= mh
    dims, lo, d2 = golden["d2"]
    want = F.relocalize_field(d2, dims, lo, RES, TR, fp, rot, t0, step, nt, K, dq, fstep, fnt)
    n, best, got, refined, status = _call_field(ctxs[0], G, fp, rot, t0, step, nt, K, True, dq, fstep, fnt)
    assert n == K == len(want["candidates"])
    _same_candidates(got, want["candidates"])
    ver = F.verify_scores(d2, dims, lo, RES, TR, fp, [(r.q_w_curr, r.t_w_curr) for r in refined])
    assert [c["verify_score"] for c in got] == ver
    per_group = len(dq) * int(np.prod(fnt))
    if name == "large group":   # a pick beyond the first 1 024-thread pass, better than everything in it
        assert per_group > TILE
        assert any(c["fine_index"] >= TILE and fs[:TILE].max() < c["fine_score"] for c, fs in zip(want["candidates"], want["fine"]))
    elif name == "one hypothesis":
        assert per_group == 1 and all(c["fine_index"] == 0 for c in got)
    elif name in ("step 0", "repeated rotations"):   # ties in every group, and the pick is the lowest of them
        for c, fs in zip(want["candidates"], want["fine"]):
            assert np.count_nonzero(fs == fs.max()) > 1 and c["fine_index"] == int(np.flatnonzero(fs == fs.max())[0])
    if mh is not None:
        G["field"].close()


# ---------------------------------------------------------------------------------------------- the shipped sizes: the C2 room at the defaults
@pytest.fixture(scope="module")
def c2(ctxs):
    from loam_livox_b200.registration import Livox_laser, Map, voxel_grid_filter
    import bench
    mc, ms = S.make_map(bench.N_MAP_CORNER, bench.N_MAP_SURF)
    truth = S.Pose(S.quat_from_euler(0.0, 0.0, np.radians(0.5)), np.array([10.05, -0.97, 0.1]))   # test_gpu_reloc_field's whole-room case
    lx = Livox_laser(ctxs[0])
    lx.extract_laser_features(S.make_scan(100000, truth, seed=S.SEED + 77), 100.0)
    c, s, _ = lx.get_features(0.0, 1.0)
    fc = voxel_grid_filter(ctxs[0], voxel_grid_filter(ctxs[0], c, 0.1), 0.2)
    fs = voxel_grid_filter(ctxs[0], voxel_grid_filter(ctxs[0], s, 0.2), 0.4)
    return mc, ms, Map(ctxs[0], mc, ms), truth, fc, fs


def test_shipped_field_search_equals_numpy(ctxs, c2):
    from loam_livox_b200.registration import RelocField, fine_search, relocalize_field, voxel_grid_filter, window_lattice, yaw_circle
    mc, ms, m, truth, fc, fs = c2
    window = ROOM + ((truth.t[2], truth.t[2], 0.0),)
    f = RelocField(ctxs[0], m, 0.2, 2, 1 << 17)
    out = relocalize_field(ctxs[0], m, f, fc, fs, window=window, yaw_step_deg=10.0, k=8)   # every default: score leaf, fine search
    sp = (voxel_grid_filter(ctxs[0], fc, 0.5), voxel_grid_filter(ctxs[0], fs, 0.5))        # the wrapper's own score points
    assert out["n_score"] == (sp[0].shape[0], sp[1].shape[0]) and sp[1].shape[0] > TILE
    rot = yaw_circle(10.0)
    t0, step, nt = window_lattice(window)
    dq, fstep, fnt = fine_search(10.0, window)
    assert len(rot) * int(np.prod(nt)) == 16236 and len(dq) * int(np.prod(fnt)) == 10571
    dims, lo, d2 = F.field([mc, ms], 0.2, 2)
    want = F.relocalize_field(d2, dims, lo, 0.2, 2, sp, rot, t0, step, nt, 8, dq, fstep, fnt)
    assert want["n_peaks"] > 8
    _same_candidates(out["candidates"], want["candidates"])
    ver = F.verify_scores(d2, dims, lo, 0.2, 2, sp, [(r.q_w_curr, r.t_w_curr) for r in out["refined"]])
    assert [c["verify_score"] for c in out["candidates"]] == ver
    ok = [j for j, r in enumerate(out["refined"]) if out["item_status"][j] == 0 and r.registered == 1 and r.status == 1]
    assert ok and out["best"] == min(ok, key=lambda j: (-ver[j], out["refined"][j].inlier_threshold, j))
    f.close()


def test_shipped_occupancy_search_equals_numpy(ctxs, c2):
    from loam_livox_b200.registration import RelocIndex, relocalize, voxel_grid_filter, window_lattice, yaw_circle
    mc, ms, m, truth, fc, fs = c2
    window = ROOM + ((truth.t[2], truth.t[2], 0.0),)
    idx = RelocIndex(ctxs[0], m, 0.2, 1, 1 << 17)
    pts = voxel_grid_filter(ctxs[0], np.concatenate([fc, fs]), 0.5)
    out = relocalize(ctxs[0], m, idx, fc, fs, window=window, yaw_step_deg=10.0, k=8)
    assert out["n_score"] == pts.shape[0] > TILE
    rot = yaw_circle(10.0)
    t0, step, nt = window_lattice(window)
    d, lo, grid = R.index([mc, ms], 0.2, 1)[:3]
    want = R.relocalize(grid, d, lo, 0.2, 1, pts, rot, t0, step, nt, 8)
    assert want["n_peaks"] > 8 and len(out["candidates"]) == 8
    _same_candidates(out["candidates"], want["candidates"], fine=False)
    ok = [j for j, r in enumerate(out["refined"]) if out["item_status"][j] == 0 and r.registered == 1 and r.status == 1]
    assert out["best"] == (min(ok, key=lambda j: (out["refined"][j].inlier_threshold, j)) if ok else -1)
    idx.close()


# ---------------------------------------------------------------------------------------------- the recovery's inputs (DESIGN.md §4.3.2)
def _qmul(a, b):
    return [a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
            a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1], a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0]]


def _yaw_quat(deg):
    a = deg * (math.pi / 180.0) * 0.5   # the library's order of operations, with the same libm
    return [math.cos(a), 0.0, 0.0, math.sin(a)]


def recovery_inputs(cfg, q, t, bad, dims, lo, n_feat, max_features):
    """§4.3.2 restated from the mapper's pose (q, t) before the step, its bad-step count, the field's grid and the step's feature count:
    (coarse rotations, t0, step, nt, fine rotations, fine step, fine nt, K)."""
    q, t = [float(v) for v in q], [float(v) for v in t]
    yaw = math.atan2(2.0 * (q[0] * q[3] + q[1] * q[2]), 1.0 - 2.0 * (q[2] * q[2] + q[3] * q[3]))
    qy = _yaw_quat(yaw * (180.0 / math.pi))
    tilt = _qmul([qy[0], -qy[1], -qy[2], -qy[3]], q)
    nn = math.sqrt(tilt[0] * tilt[0] + tilt[1] * tilt[1] + tilt[2] * tilt[2] + tilt[3] * tilt[3])
    tilt = [v / nn for v in tilt]
    n_yaw = int(math.floor(360.0 / cfg.yaw_step_deg + 0.5))   # lround of a positive value
    rot_c = np.array([_qmul(_yaw_quat(k * (360.0 / n_yaw)), tilt) for k in range(n_yaw)])
    W = cfg.window_base + cfg.window_growth * bad
    h = int(math.floor(W / cfg.t_step + 1e-9))
    i0, i1, fallback = [0, 0], [0, 0], [False, False]
    for a in range(2):
        glo = float(lo[a])
        ghi = glo + float(int(dims[a]) - 2 * cfg.trunc) * float(cfg.res)
        i0[a] = max(-h, math.ceil((glo - t[a]) / cfg.t_step))
        i1[a] = min(h, math.floor((ghi - t[a]) / cfg.t_step))
        if i0[a] > i1[a]:   # the pose off the grid on this axis: its own coordinate only
            i0[a] = i1[a] = 0
            fallback[a] = True
    max_lat = cfg.max_hypotheses // n_yaw
    trims = 0
    while (i1[0] - i0[0] + 1) * (i1[1] - i0[1] + 1) > max_lat:   # the wider axis loses its end farther from the pose
        a = 0 if (i1[0] - i0[0]) >= (i1[1] - i0[1]) else 1
        if -i0[a] > i1[a]:
            i0[a] += 1
        else:
            i1[a] -= 1
        trims += 1
    t0 = (t[0] + i0[0] * cfg.t_step, t[1] + i0[1] * cfg.t_step, t[2])
    nt = (i1[0] - i0[0] + 1, i1[1] - i0[1] + 1, 1)
    ny = int(math.floor(0.5 * cfg.yaw_step_deg / cfg.fine_yaw_step_deg + 1e-9))
    rot_f = np.array([_yaw_quat(k * cfg.fine_yaw_step_deg) for k in range(-ny, ny + 1)])
    fn = 2 * int(math.floor(cfg.fine_t_half * cfg.t_step / cfg.fine_t_step + 1e-9)) + 1
    fnt = (fn if nt[0] > 1 else 1, fn if nt[1] > 1 else 1, 1)
    K = cfg.max_candidates
    if n_feat > 0 and K * n_feat > max_features:
        K = max(1, max_features // n_feat)
    return {"rot_c": rot_c, "t0": t0, "step": (cfg.t_step,) * 3, "nt": nt, "rot_f": rot_f, "fstep": (cfg.fine_t_step,) * 3, "fnt": fnt, "K": K,
            "trims": trims, "fallback": fallback, "fine_nt": fn}


def _score_leaf(feat, leaf, oracle):
    leaf = np.float32(leaf)
    while True:
        v = oracle.voxel_grid(feat, float(leaf)) if feat.shape[0] else feat
        if v.shape[0] <= MAX_PTS:
            return v, float(leaf)
        leaf = np.float32(leaf * np.float32(2.0))


def _check_attempt(ctx, lm, cfg, e, pose_before, oracle, pipeline=True):
    """One attempt's inputs against §4.3.2 restated, its score points against the oracle's VoxelGrid, and (pipeline) the search on them against
    NumPy.  Returns the restated inputs."""
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import RelocField
    inp = lm.recovery_last_inputs()
    m = lm.whole_map()   # mode 0 searches the match map: the same clouds while every bad step is held back (nothing appended since the loss)
    f = RelocField(ctx, m, cfg.res, cfg.trunc, cfg.max_hypotheses)
    dims, lo, _ = f.read(0)
    n_feat = inp["corner"].shape[0] + inp["surf"].shape[0]
    want = recovery_inputs(cfg, *pose_before, e.bad_steps, dims, lo, n_feat, lm.ctx.cfg.max_features)
    co, fi = inp["coarse"], inp["fine"]
    assert inp["rot_coarse"].shape == want["rot_c"].shape and np.array_equal(inp["rot_coarse"], want["rot_c"]), np.abs(inp["rot_coarse"] - want["rot_c"]).max()
    assert tuple(co.t0) == want["t0"] and tuple(co.step) == want["step"] and tuple(co.nt) == want["nt"] and co.n_rot == len(want["rot_c"])
    assert co.rot_cyclic == 1 and co.max_candidates == want["K"]
    assert np.array_equal(inp["rot_fine"], want["rot_f"]) and tuple(fi.step) == want["fstep"] and tuple(fi.nt) == want["fnt"] and fi.n_rot == len(want["rot_f"])
    assert tuple(e.nt) == want["nt"] and e.n_yaw == len(want["rot_c"])
    # the score points: one VoxelGrid of each class at the score leaf, doubled until the class fits
    for cls, (feat, key) in enumerate(((inp["corner"], "score_corner"), (inp["surf"], "score_surf"))):
        v, leaf = _score_leaf(feat, cfg.score_leaf, oracle)
        assert np.float32(e.score_leaf[cls]) == np.float32(leaf) and np.array_equal(inp[key], v), (cls, leaf, e.score_leaf[cls])
    if pipeline:   # the search on these inputs: the public call's candidates are NumPy's, and the attempt is that call
        K = co.max_candidates
        cand, res, status = (capi.RelocFieldCandidate * K)(), (capi.RegResult * K)(), (C.c_int * K)()
        n, best = C.c_int(), C.c_int()
        p = [np.ascontiguousarray(inp[k]) for k in ("score_corner", "score_surf", "corner", "surf")]
        ctx.check(ctx._lib.ll_relocalize_field(ctx.h, m.h, f.h, p[0].ctypes.data, p[0].shape[0], p[1].ctypes.data, p[1].shape[0], p[2].ctypes.data, p[2].shape[0],
                                               p[3].ctypes.data, p[3].shape[0], capi.LL_FMT_XYZI16, capi.LL_HOST, C.byref(co), C.byref(fi), C.byref(inp["tmpl"]),
                                               cand, res, status, C.byref(n), C.byref(best)))
        assert (n.value, best.value) == (e.n_cand, e.best)
        _, _, d2 = f.read(0)
        d2 = [d2, f.read(1)[2]]
        w = F.relocalize_field(d2, dims, lo, cfg.res, cfg.trunc, (p[0], p[1]), want["rot_c"], want["t0"], want["step"], want["nt"], K, want["rot_f"],
                               want["fstep"], want["fnt"])
        got = [{"hypothesis": x.hypothesis, "score": x.score, "q": np.array(x.q_wxyz), "t": np.array(x.t), "fine_index": x.fine_index,
                "fine_score": x.fine_score, "fine_q": np.array(x.fine_q_wxyz), "fine_t": np.array(x.fine_t)} for x in (cand[i] for i in range(n.value))]
        _same_candidates(got, w["candidates"])
    f.close(); m.release()
    return want


def _mapper(ctx, mode, p0, pipe=None):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping
    pipe = pipe or capi.PipelineCfg(pieces=3, use_piece=0, extractor_leaf_corner=0.1, extractor_leaf_surf=0.2, mapping_leaf_corner=0.1, mapping_leaf_surf=0.4,
                                    whole_frame=1)
    st = capi.default_reg_state(mapping_init_accumulate_frames=3, q_w_last=p0.q, t_w_last=p0.t, q_w_curr=p0.q, t_w_curr=p0.t)
    return Laser_mapping(ctx, reg=st, pipeline=pipe, matching_mode=mode, maximum_history_size=400)


K_JUMP = 160   # tests/test_gpu_recovery.py's kidnap: 1 m back, 2 m aside, 15 deg, from scan 160 on


@pytest.fixture(scope="module")
def kidnap_stream():
    poses = S.trajectory(n_scans=K_JUMP + 12, n_static=4, speed=1.0)
    kid = lambda p: S.Pose(S.quat_mul(p.q, S.quat_from_euler(0.0, 0.0, np.radians(-15.0))), p.t + np.array([-1.0, -2.0, 0.0]))  # noqa: E731
    poses = poses[:K_JUMP] + [kid(p) for p in poses[K_JUMP:]]
    seed = S.SEED + 2300
    return poses, [S.make_scan(24000, p, seed=seed + k) for k, p in enumerate(poses)], [100.0 + 0.1 * k for k in range(len(poses))]


@pytest.mark.parametrize("mode", [0, 1])
def test_recovery_inputs_in_the_kidnap(ctxs, kidnap_stream, oracle, mode):
    poses, raws, stamps = kidnap_stream
    lm = _mapper(ctxs[0], mode, poses[0])
    cfg = lm.set_recovery()
    n_att = 0
    for k in range(len(raws)):
        before = lm.pose()[:2]
        lm.process_new_scan(raws[k], stamps[k])
        log, _ = lm.recovery_log()
        if log and log[-1].attempted:
            assert log[-1].attempt_status == 0
            _check_attempt(ctxs[1], lm, cfg, log[-1], before, oracle)
            n_att += 1
    assert n_att >= 1
    lm.close()


@pytest.fixture(scope="module")
def short_stream():
    poses = S.trajectory(n_scans=12, n_static=4, speed=1.0)
    return poses, [S.make_scan(24000, p, seed=S.SEED + 3100 + k) for k, p in enumerate(poses)], [100.0 + 0.1 * k for k in range(len(poses))]


BRANCHES = {
    "shrink": dict(max_hypotheses=36 * 12, window_base=4.0, fine_t_half=0.0),   # 36 yaws x the window > max_hypotheses; fine nt 1 on every axis
    "K lowered": dict(max_candidates=16),                       # 16 x the step's features > max_features (a context of 16 000)
    "one-point axes": dict(window_base=0.0, window_growth=0.0),  # a window of 0 steps: coarse nt 1 on x and y, so fine nt 1 there too
    "off the grid": dict(window_base=1.0, window_growth=0.0),    # the pose moved 1.5 steps below the grid in x: x is the pose's own
}


@pytest.mark.parametrize("branch", list(BRANCHES))
@pytest.mark.parametrize("mode", [0, 1])
def test_recovery_inputs_on_other_branches(ctxs, short_stream, oracle, branch, mode):
    """Every step held back from scan 6 on (max_inlier_threshold 0), so every step from the third on attempts."""
    from loam_livox_b200.registration import Context
    poses, raws, stamps = short_stream
    ctx = Context(0, max_scan_points=60000, max_features=16000) if branch == "K lowered" else ctxs[0]
    lm = _mapper(ctx, mode, poses[0])
    for k in range(6):
        lm.process_new_scan(raws[k], stamps[k])
    cfg = lm.set_recovery(max_inlier_threshold=0.0, **BRANCHES[branch])
    if branch == "off the grid":   # just past the map's bounding box, so the step still registers (floor and ceiling) but the window misses x
        from loam_livox_b200.registration import RelocField
        m = lm.whole_map()
        f = RelocField(ctxs[1], m, cfg.res, cfg.trunc, cfg.max_hypotheses)
        _, lo, _ = f.read(0)
        f.close(); m.release()
        q, t, _ = lm.pose()
        lm.set_pose(q, np.array([float(lo[0]) - 1.5 * cfg.t_step, t[1], t[2]]))
    n_att = 0
    for k in range(6, len(raws)):
        before = lm.pose()[:2]
        lm.process_new_scan(raws[k], stamps[k])
        log, _ = lm.recovery_log()
        if log[-1].attempted:
            assert log[-1].attempt_status == 0
            want = _check_attempt(ctxs[1], lm, cfg, log[-1], before, oracle, pipeline=n_att == 0)
            n_att += 1
            if branch == "shrink":   # the loop ran and left the window off-centre
                assert want["trims"] >= 2 and want["nt"][0] * want["nt"][1] <= 12 and want["fnt"] == (1, 1, 1), (want["nt"], want["trims"], log[-1].bad_steps)
            elif branch == "K lowered":
                assert want["K"] < cfg.max_candidates
            elif branch == "one-point axes":
                assert want["nt"] == (1, 1, 1) and want["fine_nt"] > 1 and want["fnt"] == (1, 1, 1)
            elif branch == "off the grid":
                assert want["fallback"] == [True, False] and want["t0"][0] == before[1][0] and want["nt"][0] == 1 and want["nt"][1] > 1
                assert want["fine_nt"] > 1 and want["fnt"] == (1, want["fine_nt"], 1)
    assert n_att >= 4
    lm.close()
    if ctx is not ctxs[0]:
        ctx.close()


def test_recovery_score_leaf_doubled_more_than_once(ctxs, oracle):
    """Scans dense enough that a class of the step's features keeps more than 8 192 points at twice the score leaf."""
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Context
    ctx = Context(0, max_scan_points=200000, max_features=200000)
    poses = S.trajectory(n_scans=9, n_static=4, speed=1.0)
    raws = [S.make_scan(150000, p, seed=S.SEED + 3300 + k) for k, p in enumerate(poses)]
    pipe = capi.PipelineCfg(pieces=3, use_piece=0, extractor_leaf_corner=0.02, extractor_leaf_surf=0.02, mapping_leaf_corner=0.02, mapping_leaf_surf=0.02,
                            whole_frame=1)
    lm = _mapper(ctx, 0, poses[0], pipe)
    for k in range(5):
        lm.process_new_scan(raws[k], 100.0 + 0.1 * k)
    cfg = lm.set_recovery(max_inlier_threshold=0.0, score_leaf=0.01)
    n_att = 0
    for k in range(5, len(raws)):
        before = lm.pose()[:2]
        lm.process_new_scan(raws[k], 100.0 + 0.1 * k)
        log, _ = lm.recovery_log()
        if log[-1].attempted:
            assert log[-1].attempt_status == 0
            _check_attempt(ctxs[1], lm, cfg, log[-1], before, oracle, pipeline=False)
            assert max(log[-1].score_leaf) >= 4 * np.float32(0.01)
            n_att += 1
    assert n_att >= 1
    lm.close(); ctx.close()
