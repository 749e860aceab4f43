"""Relocalization by class-aware distance fields on the GPU (ll_reloc_field_build, ll_reloc_field_scores, ll_relocalize_field): the fields and
the scores equal the NumPy restatement (tests/reloc_field_reference.py) byte for byte and integer for integer, the candidates, fine picks and verify
scores of one call are NumPy's, every refined item is ll_register_batch from the same seeds, a scan of the C2 room is found over the whole room
(also off the lattice), and a saved mapper restarts there from a 1 m lattice."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from loam_livox_b200 import synthetic as S  # noqa: E402
import reloc_field_reference as F  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "golden_small.npz")
ROOM = ((-1.0, 39.0, 1.0), (-5.0, 5.0, 1.0))


@pytest.fixture(scope="module")
def ctxs():
    from loam_livox_b200.registration import Context
    a = Context(0, max_scan_points=200000, max_features=400000)
    b = Context(0, max_scan_points=200000, max_features=400000)
    yield a, b
    a.close(); b.close()


@pytest.fixture(scope="module")
def c2(ctxs):
    from loam_livox_b200.registration import Map
    import bench
    mc, ms = S.make_map(bench.N_MAP_CORNER, bench.N_MAP_SURF)
    return mc, ms, Map(ctxs[0], mc, ms)


def _result_key(r):
    from loam_livox_b200 import capi
    return tuple(np.array(list(getattr(r, f)) if isinstance(getattr(r, f), C.Array) else [getattr(r, f)]).tobytes()
                 for f, _ in capi.RegResult._fields_ if not f.startswith("gpu_ms"))


def _check_field(ctx, m, clouds, res, T):
    from loam_livox_b200.registration import RelocField
    f = RelocField(ctx, m, res, T, 1024)
    dims, lo, d2 = F.field(clouds, res, T)
    for which in (0, 1):
        gd, glo, g = f.read(which)
        assert gd.tolist() == dims.tolist() and np.array_equal(glo, lo)
        assert np.array_equal(g, d2[which]), (res, T, which)
    return f, (dims, lo, d2)


# ---------------------------------------------------------------------------------------------- the fields
def test_field_golden_small(ctxs):
    from loam_livox_b200.registration import Map
    g = np.load(GOLDEN)
    m = Map(ctxs[0], g["map_corner"], g["map_surf"])
    for res, T in ((0.3, 1), (0.5, 5), (0.25, 15)):
        _check_field(ctxs[0], m, [g["map_corner"], g["map_surf"]], res, T)[0].close()


@pytest.mark.parametrize("res", [0.2, 0.3])
@pytest.mark.parametrize("T", [1, 5, 15])
def test_field_c2_map(ctxs, c2, res, T):
    mc, ms, m = c2
    _check_field(ctxs[0], m, [mc, ms], res, T)[0].close()


def test_field_one_point_at_negative_coordinates_and_an_empty_class(ctxs):
    from loam_livox_b200.registration import Map
    one = np.array([[-3.5, 2.25, -0.125, 0]], np.float32)
    m1 = Map(ctxs[0], one, one)
    f, (dims, _, d2) = _check_field(ctxs[0], m1, [one, one], 0.5, 3)
    assert dims.tolist() == [7, 7, 7] and d2[0][3, 3, 3] == 0 and d2[0][0, 0, 0] == 9   # (3^2 + 3^2 + 3^2 clamped)
    f.close()
    nan = np.array([[np.nan, np.nan, np.nan, 0]], np.float32)   # a class without a finite point: T^2 everywhere
    surf = np.array([[-1.0, -2.0, -0.5, 0], [0.5, 0.25, 1.0, 0], [-0.25, -1.75, -0.25, 0]], np.float32)
    m2 = Map(ctxs[0], nan, surf)
    f, (_, _, d2) = _check_field(ctxs[0], m2, [nan, surf], 0.25, 5)
    assert (d2[0] == 25).all() and (d2[1] == 0).sum() == 3
    f.close()


# ---------------------------------------------------------------------------------------------- scores, candidates, picks, refinement, verify
def _golden_case(ctx, res=0.3, T=5, max_hyp=4096):
    from loam_livox_b200.registration import Map, RelocField, voxel_grid_filter
    g = np.load(GOLDEN)
    m = Map(ctx, g["map_corner"], g["map_surf"])
    f = RelocField(ctx, m, res, T, max_hyp)
    pts = (voxel_grid_filter(ctx, g["feat_corner"], 0.3), voxel_grid_filter(ctx, g["feat_surf"], 0.3))
    return g, m, f, pts


def _yaws(deg):
    a = np.radians(np.asarray(deg, np.float64)) * 0.5
    return np.stack([np.cos(a), 0 * a, 0 * a, np.sin(a)], axis=1)


def test_field_scores_equal_numpy(ctxs):
    from loam_livox_b200.registration import reloc_field_scores
    g, m, f, pts = _golden_case(ctxs[0])
    dims, lo, d2 = F.field([g["map_corner"], g["map_surf"]], 0.3, 5)
    bad = np.float32([[np.nan, 1, 1, 0], [0, 0, 0, 0], [1, np.inf, 0, 0]])
    sp = (np.concatenate([pts[0], bad]), np.concatenate([pts[1], bad[::-1]]))
    tilt = S.quat_from_euler(0.03, -0.02, 0.0)
    rot = np.array([S.quat_mul(q, tilt) for q in _yaws([0.0, 7.0, -12.0, 180.0])])
    t = g["guess_t"]
    cases = [(rot, (t[0] - 6.0, t[1] - 2.0, t[2] - 0.3), (1.5, 1.0, 0.3), (9, 5, 3)),     # far steps push points out of the grid
             (rot[:1], tuple(t), (1.0, 1.0, 1.0), (1, 1, 1))]                              # one rotation, one translation
    for rr, t0, step, nt in cases:
        got = reloc_field_scores(ctxs[0], f, sp[0], sp[1], rr, t0, step, nt)
        want = F.field_scores(d2, dims, lo, 0.3, 5, sp, rr, t0, step, nt)
        assert got.dtype == np.int32 and np.array_equal(got, want)
    assert want.max() > 0
    f.close()


def test_one_call_equals_numpy_and_the_batch(ctxs):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import fine_search, register_batch, relocalize_field, window_lattice, yaw_circle
    g, m, f, pts = _golden_case(ctxs[0])
    dims, lo, d2 = F.field([g["map_corner"], g["map_surf"]], 0.3, 5)
    fc, fs = np.ascontiguousarray(g["feat_corner"], np.float32), np.ascontiguousarray(g["feat_surf"], np.float32)
    t = g["guess_t"]
    window = ((t[0] - 0.6, t[0] + 0.6, 0.3), (t[1] - 0.6, t[1] + 0.6, 0.3), (t[2], t[2], 0.0))
    out = relocalize_field(ctxs[0], m, f, fc, fs, window=window, yaw_step_deg=5.0, k=6, score_pts=pts, fine_yaw_step_deg=1.0, fine_t_step=0.05,
                           fine_t_half=0.5)
    rot = yaw_circle(5.0)
    t0, step, nt = window_lattice(window)
    dq, fstep, fnt = fine_search(5.0, window, 1.0, 0.05, 0.5)
    want = F.relocalize_field(d2, dims, lo, 0.3, 5, pts, rot, t0, step, nt, 6, dq, fstep, fnt)["candidates"]
    assert len(out["candidates"]) == len(want) > 1
    for c, w in zip(out["candidates"], want):
        assert (c["hypothesis"], c["score"], c["fine_index"], c["fine_score"]) == (w["hypothesis"], w["score"], w["fine_index"], w["fine_score"])
        assert all(np.array_equal(c[k], w[k]) for k in ("q", "t", "fine_q", "fine_t"))
    # the refined items: one ll_register_batch from the same seeds on another context
    state0 = capi.default_reg_state()
    state0.current_frame_index = state0.mapping_init_accumulate_frames + 1
    seeds = [capi.default_reg_state(q_w_last=c["fine_q"], t_w_last=c["fine_t"], q_w_curr=c["fine_q"], t_w_curr=c["fine_t"],
                                    current_frame_index=state0.current_frame_index) for c in out["candidates"]]
    res, status = register_batch(ctxs[1], m, [(fc, fs)] * len(seeds), seeds)
    assert status == out["item_status"]
    assert [_result_key(r) for r in res] == [_result_key(r) for r in out["refined"]]
    # verify scores at the refined poses, and the choice
    ver = [int(F.field_scores(d2, dims, lo, 0.3, 5, pts, np.array(r.q_w_curr)[None], tuple(r.t_w_curr), (0.0, 0.0, 0.0), (1, 1, 1))[0]) for r in out["refined"]]
    assert [c["verify_score"] for c in out["candidates"]] == ver
    ok = [j for j, r in enumerate(out["refined"]) if out["item_status"][j] == 0 and r.registered == 1 and r.status == 1]
    assert ok
    assert out["best"] == min(ok, key=lambda j: (-ver[j], out["refined"][j].inlier_threshold, j))
    f.close()


def test_two_contexts_give_identical_outputs(ctxs):
    from loam_livox_b200.registration import relocalize_field
    outs = []
    for ctx in ctxs:
        g, m, f, pts = _golden_case(ctx)
        t = g["guess_t"]
        window = ((t[0] - 0.9, t[0] + 0.9, 0.3), (t[1] - 0.9, t[1] + 0.9, 0.3), (t[2], t[2], 0.0))
        o = relocalize_field(ctx, m, f, g["feat_corner"], g["feat_surf"], window=window, yaw_step_deg=10.0, k=8, score_pts=pts, fine_t_half=0.5)
        outs.append(([{k: np.asarray(v).tobytes() for k, v in c.items()} for c in o["candidates"]], [_result_key(r) for r in o["refined"]], o["item_status"], o["best"]))
        f.close()
    assert outs[0] == outs[1] and len(outs[0][0]) > 0


# ---------------------------------------------------------------------------------------------- end to end in the C2 room
def _c2_features(ctx, pose, n=100000, seed=S.SEED + 77):
    from loam_livox_b200.registration import Livox_laser, voxel_grid_filter
    lx = Livox_laser(ctx)
    lx.extract_laser_features(S.make_scan(n, pose, seed=seed), 100.0)
    c, s, _ = lx.get_features(0.0, 1.0)
    return voxel_grid_filter(ctx, voxel_grid_filter(ctx, c, 0.1), 0.2), voxel_grid_filter(ctx, voxel_grid_filter(ctx, s, 0.2), 0.4)


@pytest.mark.parametrize("x,y,yaw_deg", [(10.05, -0.97, 0.5),    # the pose tests/test_gpu_relocalize.py finds in a one-pitch window
                                         (10.55, -0.47, 5.5)])   # off the lattice: about 0.65 m and 4.5 deg from the nearest hypothesis
def test_end_to_end_c2_whole_room(ctxs, c2, x, y, yaw_deg):
    from loam_livox_b200.registration import RelocField, relocalize_field
    mc, ms, m = c2
    truth = S.Pose(S.quat_from_euler(0.0, 0.0, np.radians(yaw_deg)), np.array([x, y, 0.1]))
    fc, fs = _c2_features(ctxs[0], truth)
    f = RelocField(ctxs[0], m, 0.2, 2, 1 << 17)
    out = relocalize_field(ctxs[0], m, f, fc, fs, window=ROOM + ((truth.t[2], truth.t[2], 0.0),), yaw_step_deg=10.0, k=8)
    b = out["best"]
    assert b >= 0, out["candidates"]
    r = out["refined"][b]
    err_t, err_r = np.linalg.norm(np.array(r.t_w_curr) - truth.t), np.degrees(S.quat_angle(np.array(r.q_w_curr), truth.q))
    assert err_t < 0.05 and err_r < 0.5, (err_t, err_r, [(c["t"].tolist(), c["verify_score"]) for c in out["candidates"]])
    f.close()


# ---------------------------------------------------------------------------------------------- the streaming mapper
def _mapper(ctx, mode, init=3, window=400, **reg):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping
    pipe = capi.PipelineCfg(pieces=3, use_piece=0, extractor_leaf_corner=0.1, extractor_leaf_surf=0.2, mapping_leaf_corner=0.1, mapping_leaf_surf=0.4, whole_frame=1)
    return Laser_mapping(ctx, reg=capi.default_reg_state(mapping_init_accumulate_frames=init, **reg), pipeline=pipe, matching_mode=mode, maximum_history_size=window)


@pytest.mark.parametrize("mode", [0, 1])
def test_session_restart_from_a_one_metre_lattice(ctxs, mode):
    """Save at scan k0, load on a fresh context, relocalize scan k0 + 20 from a 1 m lattice and 10 deg yaws, set the pose and go on for 10 scans:
    every scan accepted, every pose within 0.05 m / 0.5 deg of the synthetic truth beyond the error of the mapper that ran the whole stream."""
    from loam_livox_b200.registration import Context, Laser_mapping, Livox_laser, RelocField, relocalize_field, voxel_grid_filter
    k0 = 12
    poses = S.trajectory(n_scans=k0 + 31, n_static=4, speed=1.0)
    raws = [S.make_scan(24000, p, seed=S.SEED + 1300 + k) for k, p in enumerate(poses)]
    stamps = [100.0 + 0.1 * k for k in range(k0 + 31)]
    p0 = poses[0]
    gm = _mapper(ctxs[0], mode, q_w_last=p0.q, t_w_last=p0.t, q_w_curr=p0.q, t_w_curr=p0.t)
    ref = {}
    for k in range(k0 + 30):
        gm.process_new_scan(raws[k], stamps[k])
        if k == k0:
            img = gm.save()
        ref[k] = gm.pose()[:2]
    gm.close()
    ctx = Context(0, max_scan_points=60000, max_features=60000)
    lm = Laser_mapping.load(ctx, img)
    m = lm.whole_map()
    f = RelocField(ctx, m, 0.2, 2, 1 << 17)
    k = k0 + 20
    lx = Livox_laser(ctx)
    lx.extract_laser_features(raws[k], stamps[k])
    c, s, _ = lx.get_features(0.0, 1.0)
    fc = voxel_grid_filter(ctx, voxel_grid_filter(ctx, c, 0.1), 0.1)
    fs = voxel_grid_filter(ctx, voxel_grid_filter(ctx, s, 0.2), 0.4)
    out = relocalize_field(ctx, m, f, fc, fs, score_leaf=0.3, window=((-1.0, 3.0, 1.0), (-2.0, 2.0, 1.0), (poses[k].t[2], poses[k].t[2], 0.0)),
                           yaw_step_deg=10.0, k=8)
    assert out["best"] >= 0
    r = out["refined"][out["best"]]
    lm.set_pose(np.array(r.q_w_curr), np.array(r.t_w_curr))
    for j in range(k, k + 10):
        res, _ = lm.process_new_scan(raws[j], stamps[j])
        q, t, _ = lm.pose()
        qr, tr = ref[j]
        e_t, e_r = np.linalg.norm(t - poses[j].t), np.degrees(S.quat_angle(q, poses[j].q))
        f_t, f_r = np.linalg.norm(tr - poses[j].t), np.degrees(S.quat_angle(qr, poses[j].q))
        assert res.status == 1 and e_t < f_t + 0.05 and e_r < f_r + 0.5, (j, t, tr, poses[j].t)
    f.close(); m.release(); lm.close(); ctx.close()


# ---------------------------------------------------------------------------------------------- validation
def _raw_call(ctx, m, f, sp, fc, fs, coarse, fine, st, K=16):
    from loam_livox_b200 import capi
    cand, res, status = (capi.RelocFieldCandidate * K)(), (capi.RegResult * K)(), (C.c_int * K)()
    n, best = C.c_int(), C.c_int()
    rc = ctx._lib.ll_relocalize_field(ctx.h, m.h if m else None, f.h if f else None, sp[0].ctypes.data, sp[0].shape[0], sp[1].ctypes.data, sp[1].shape[0],
                                      fc.ctypes.data, fc.shape[0], fs.ctypes.data, fs.shape[0], capi.LL_FMT_XYZI16, capi.LL_HOST,
                                      C.byref(coarse) if coarse is not None else None, C.byref(fine) if fine is not None else None, C.byref(st),
                                      cand, res, status, C.byref(n), C.byref(best))
    val = lambda x: np.array(list(x) if isinstance(x, C.Array) else [x]).tobytes()  # noqa: E731
    key = [tuple(val(getattr(cand[i], fl)) for fl, _ in capi.RelocFieldCandidate._fields_) + _result_key(res[i]) + (status[i],) for i in range(n.value)]
    return rc, key, best.value


def test_validation_leaves_the_context_usable(ctxs):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Context, Map, fine_cfg, reloc_cfg, yaw_circle
    ctx = ctxs[0]
    g, m, f, pts = _golden_case(ctx)
    fc, fs = np.ascontiguousarray(g["feat_corner"], np.float32), np.ascontiguousarray(g["feat_surf"], np.float32)
    t = g["guess_t"]
    rot = yaw_circle(30.0)
    good, _k1 = reloc_cfg(rot, (t[0] - 0.3, t[1] - 0.3, t[2]), (0.3, 0.3, 1.0), (3, 3, 1), k=4)
    dq = _yaws([-2.0, 0.0, 2.0])
    fine, _k2 = fine_cfg(dq, (0.1, 0.1, 0.1), (3, 3, 1))
    st = capi.default_reg_state(current_frame_index=51, mapping_init_accumulate_frames=50)
    L = ctx._lib
    # the field build
    h = C.c_void_p()
    for res, T, mh, code in ((0.0, 5, 10, capi.LL_ERR_INVALID), (-1.0, 5, 10, capi.LL_ERR_INVALID), (float("nan"), 5, 10, capi.LL_ERR_INVALID),
                             (0.3, 0, 10, capi.LL_ERR_INVALID), (0.3, 16, 10, capi.LL_ERR_INVALID), (0.3, 5, 0, capi.LL_ERR_INVALID),
                             (0.3, 5, (1 << 24) + 1, capi.LL_ERR_INVALID), (1e-4, 5, 10, capi.LL_ERR_CAPACITY)):
        assert L.ll_reloc_field_build(ctx.h, m.h, res, T, mh, C.byref(h)) == code, (res, T, mh)
        assert not h.value
    sharded = Map(ctx, g["map_corner"], g["map_surf"], rank=0, world=2)
    assert L.ll_reloc_field_build(ctx.h, sharded.h, 0.3, 5, 10, C.byref(h)) == capi.LL_ERR_INVALID
    # the relocalization
    bad_q = rot.copy(); bad_q[1] *= 1.001
    bad_dq = dq.copy(); bad_dq[2] *= 0.999
    none = C.POINTER(C.c_double)()
    cases = {
        "non-unit": (reloc_cfg(bad_q, good.t0, good.step, good.nt, 4)[0], fine, capi.LL_ERR_INVALID),
        "nt 0": (reloc_cfg(rot, good.t0, good.step, (3, 0, 1), 4)[0], fine, capi.LL_ERR_INVALID),
        "n_rot 0": (reloc_cfg(rot[:0], good.t0, good.step, good.nt, 4)[0], fine, capi.LL_ERR_INVALID),
        "hypotheses": (reloc_cfg(rot, good.t0, good.step, (20, 20, 1), 4)[0], fine, capi.LL_ERR_INVALID),   # 12 x 400 > 4096
        "K 0": (reloc_cfg(rot, good.t0, good.step, good.nt, 0)[0], fine, capi.LL_ERR_INVALID),
        "K 17": (reloc_cfg(rot, good.t0, good.step, good.nt, 17)[0], fine, capi.LL_ERR_INVALID),
        "no coarse": (None, fine, capi.LL_ERR_INVALID),
        "no fine": (good, None, capi.LL_ERR_INVALID),
        "fine null rotations": (good, capi.RelocFineCfg(3, none, (0.1, 0.1, 0.1), (3, 3, 1)), capi.LL_ERR_INVALID),
        "fine n_rot 0": (good, fine_cfg(dq[:0], (0.1, 0.1, 0.1), (3, 3, 1))[0], capi.LL_ERR_INVALID),
        "fine nt 0": (good, fine_cfg(dq, (0.1, 0.1, 0.1), (3, 0, 1))[0], capi.LL_ERR_INVALID),
        "fine nt even": (good, fine_cfg(dq, (0.1, 0.1, 0.1), (3, 4, 1))[0], capi.LL_ERR_INVALID),
        "fine step inf": (good, fine_cfg(dq, (0.1, float("inf"), 0.1), (3, 3, 1))[0], capi.LL_ERR_INVALID),
        "fine non-unit": (good, fine_cfg(bad_dq, (0.1, 0.1, 0.1), (3, 3, 1))[0], capi.LL_ERR_INVALID),
        "K x fine": (good, fine_cfg(dq, (0.1, 0.1, 0.1), (21, 21, 1))[0], capi.LL_ERR_INVALID),               # 4 x 3 x 441 > 4096
    }
    keep = [_k1, _k2, dq, bad_dq, bad_q]
    for name, (co, fi, code) in cases.items():
        keep.append((co, fi))
        assert _raw_call(ctx, m, f, pts, fc, fs, co, fi, st)[0] == code, name
    gated = capi.default_reg_state(current_frame_index=50, mapping_init_accumulate_frames=50)
    assert _raw_call(ctx, m, f, pts, fc, fs, good, fine, gated)[0] == capi.LL_ERR_INVALID
    other = Map(ctx, g["map_corner"], g["map_surf"])
    assert _raw_call(ctx, other, f, pts, fc, fs, good, fine, st)[0] == capi.LL_ERR_INVALID
    assert _raw_call(ctx, sharded, f, pts, fc, fs, good, fine, st)[0] == capi.LL_ERR_INVALID
    assert _raw_call(ctx, m, None, pts, fc, fs, good, fine, st)[0] == capi.LL_ERR_INVALID
    many = np.zeros((capi.LL_RELOC_MAX_SCORE_POINTS + 1, 4), np.float32)
    assert _raw_call(ctx, m, f, (many, pts[1]), fc, fs, good, fine, st)[0] == capi.LL_ERR_CAPACITY
    assert _raw_call(ctx, m, f, (pts[0], many), fc, fs, good, fine, st)[0] == capi.LL_ERR_CAPACITY
    big_fc = np.ascontiguousarray(np.tile(fc, (200, 1)))
    big_fs = np.ascontiguousarray(np.tile(fs, (200, 1)))
    assert 4 * (big_fc.shape[0] + big_fs.shape[0]) > ctx.cfg.max_features
    assert _raw_call(ctx, m, f, pts, big_fc, big_fs, good, fine, st)[0] == capi.LL_ERR_CAPACITY
    # the parity hooks
    sc = np.zeros(200, np.int32)
    assert L.ll_reloc_field_scores(ctx.h, f.h, many.ctypes.data, many.shape[0], pts[1].ctypes.data, pts[1].shape[0], capi.LL_FMT_XYZI16, capi.LL_HOST,
                                   C.byref(good), sc.ctypes.data) == capi.LL_ERR_CAPACITY
    assert L.ll_reloc_field_read(f.h, 2, None, None, None, 0) == capi.LL_ERR_INVALID
    assert L.ll_reloc_field_read(f.h, 0, None, None, sc.ctypes.data, 1) == capi.LL_ERR_CAPACITY
    # usable afterwards: the next call is a fresh context's
    rc, key, best = _raw_call(ctx, m, f, pts, fc, fs, good, fine, st)
    fresh = Context(0, max_scan_points=200000, max_features=400000)
    rc2, key2, best2 = _raw_call(fresh, m, f, pts, fc, fs, good, fine, st)
    assert rc == rc2 == capi.LL_OK and key == key2 and best == best2 and len(key) > 0
    fresh.close(); f.close()
