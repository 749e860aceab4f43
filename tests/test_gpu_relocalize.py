"""Relocalization on the GPU (ll_reloc_index_build, ll_reloc_scores, ll_relocalize, ll_mapper_whole_map, ll_mapper_set_pose): the index and the
scores equal the NumPy restatement (tests/reloc_reference.py) word for word and integer for integer, the candidates are its first K peaks, every
refined item is ll_register from that candidate's seed, a scan of the C2 room is found without a guess, and a saved mapper restarts there."""
import ctypes as C
import os
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from loam_livox_b200 import synthetic as S  # noqa: E402
import reloc_reference as R  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "golden_small.npz")
INT_FIELDS = ("status", "registered", "icp_iterations", "num_residual_blocks", "corner_used", "surf_used", "total_lm_iterations", "total_evaluations")
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


def _yaws(deg):
    a = np.radians(np.asarray(deg, np.float64)) * 0.5
    return np.stack([np.cos(a), 0 * a, 0 * a, np.sin(a)], axis=1)


def _check_index(ctx, m, clouds, res, dilate):
    from loam_livox_b200.registration import RelocIndex
    idx = RelocIndex(ctx, m, res, dilate, 1024)
    dims, lo, words = idx.read()
    d2, lo2, g, w2 = R.index(clouds, res, dilate)
    assert dims.tolist() == d2.tolist() and np.array_equal(lo, lo2)
    assert np.array_equal(words, w2)
    return idx, (d2, lo2, g)


# ---------------------------------------------------------------------------------------------- the index
def test_index_golden_small(ctxs):
    from loam_livox_b200.registration import Map
    g = np.load(GOLDEN)
    m = Map(ctxs[0], g["map_corner"], g["map_surf"])
    for res, dilate in ((0.3, 0), (0.5, 1), (0.25, 4)):
        _check_index(ctxs[0], m, [g["map_corner"], g["map_surf"]], res, dilate)[0].close()


@pytest.mark.parametrize("res,dilate", [(0.2, 1), (0.5, 2)])
def test_index_c2_map(ctxs, c2, res, dilate):
    mc, ms, m = c2
    _check_index(ctxs[0], m, [mc, ms], res, dilate)[0].close()


def test_index_faces_negative_one_point(ctxs):
    from loam_livox_b200.registration import Map
    res = 0.25
    face = np.array([[-1.0, -2.0, -0.5, 0], [-0.75, -2.0, -0.5, 0], [-0.5, -1.5, 0.0, 0], [0.5, 0.25, 1.0, 0], [-0.25, -1.75, -0.25, 0]], np.float32)
    surf = np.concatenate([face, face + np.float32([0.25, 0.5, 0.75, 0])] * 10, axis=0)
    m = Map(ctxs[0], face, surf)
    _check_index(ctxs[0], m, [face, surf], res, 2)[0].close()
    one = np.array([[-3.5, 2.25, -0.125, 0]], np.float32)
    m1 = Map(ctxs[0], one, one)
    idx, (dims, _, g) = _check_index(ctxs[0], m1, [one, one], 0.5, 3)
    assert dims.tolist() == [7, 7, 7] and g.all()   # the one voxel dilated to the whole grid, border clipped
    idx.close()


# ---------------------------------------------------------------------------------------------- scores, peaks, refinement
def _golden_case(ctx):
    from loam_livox_b200.registration import Map, RelocIndex, voxel_grid_filter
    g = np.load(GOLDEN)
    m = Map(ctx, g["map_corner"], g["map_surf"])
    idx = RelocIndex(ctx, m, 0.3, 1, 4096)
    pts = voxel_grid_filter(ctx, np.concatenate([g["feat_corner"], g["feat_surf"]]), 0.3)
    return g, m, idx, pts


def test_scores_equal_numpy(ctxs):
    from loam_livox_b200.registration import reloc_scores
    g, m, idx, pts = _golden_case(ctxs[0])
    d, lo, grid = R.index([g["map_corner"], g["map_surf"]], 0.3, 1)[:3]
    sp = np.concatenate([pts, np.float32([[np.nan, 1, 1, 0], [0, 0, 0, 0], [1, np.inf, 0, 0]])])
    tilt = S.quat_from_euler(0.03, -0.02, 0.0)
    rot = np.array([S.quat_mul(q, tilt) for q in _yaws([0.0, 7.0, -12.0, 180.0])])
    t = g["guess_t"]
    cases = [(rot, (t[0] - 6.0, t[1] - 2.0, t[2] - 0.3), (1.5, 1.0, 0.3), (9, 5, 3)),     # far steps push points out of the grid
             (rot[:1], tuple(t), (1.0, 1.0, 1.0), (1, 1, 1))]                              # one rotation, one translation
    for rr, t0, step, nt in cases:
        got = reloc_scores(ctxs[0], idx, sp, rr, t0, step, nt)
        want = R.scores(grid, d, lo, 0.3, 1, sp, rr, t0, step, nt)
        assert got.dtype == np.int32 and np.array_equal(got, want)
    assert want.max() > 0
    idx.close()


def _single(ctx, m, fc, fs, state):
    from loam_livox_b200 import capi
    res = capi.RegResult()
    st = ctx._lib.ll_register(ctx.h, m.h, fc.ctypes.data, fc.shape[0], fs.ctypes.data, fs.shape[0], capi.LL_FMT_XYZI16, capi.LL_HOST, C.byref(state), C.byref(res))
    return st, res


def test_candidates_are_numpy_peaks_and_items_are_single_registrations(ctxs, oracle):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import relocalize
    g, m, idx, pts = _golden_case(ctxs[0])
    d, lo, grid = R.index([g["map_corner"], g["map_surf"]], 0.3, 1)[:3]
    fc, fs = np.ascontiguousarray(g["feat_corner"], np.float32), np.ascontiguousarray(g["feat_surf"], np.float32)
    t = g["guess_t"]
    window = ((t[0] - 0.6, t[0] + 0.6, 0.3), (t[1] - 0.6, t[1] + 0.6, 0.3), (t[2], t[2], 0.0))
    out = relocalize(ctxs[0], m, idx, fc, fs, window=window, yaw_step_deg=5.0, k=6, score_pts=pts)
    from loam_livox_b200.registration import window_lattice, yaw_circle
    rot = yaw_circle(5.0)
    t0, step, nt = window_lattice(window)
    sc = R.scores(grid, d, lo, 0.3, 1, pts, rot, t0, step, nt)
    hs, ss = R.peaks(sc, rot.shape[0], nt, True)
    K = min(6, hs.shape[0])
    assert [c["hypothesis"] for c in out["candidates"]] == hs[:K].tolist() and [c["score"] for c in out["candidates"]] == ss[:K].tolist()
    state0 = capi.default_reg_state()
    state0.current_frame_index = state0.mapping_init_accumulate_frames + 1
    trees = (oracle.KdTree(g["map_corner"]), oracle.KdTree(g["map_surf"]))
    for j, c in enumerate(out["candidates"]):
        q, tt = R.candidate_pose(c["hypothesis"], rot, t0, step, nt)
        assert np.array_equal(c["q"], q) and np.array_equal(c["t"], tt)
        st = capi.default_reg_state(q_w_last=q, t_w_last=tt, q_w_curr=q, t_w_curr=tt, current_frame_index=state0.current_frame_index)
        st1, r1 = _single(ctxs[1], m, fc, fs, st)
        r = out["refined"][j]
        assert out["item_status"][j] == st1
        assert tuple(getattr(r, f) for f in INT_FIELDS) == tuple(getattr(r1, f) for f in INT_FIELDS), j
        assert np.abs(np.array(r.t_w_curr) - np.array(r1.t_w_curr)).max() <= 1e-9 and np.abs(np.array(r.q_w_curr) - np.array(r1.q_w_curr)).max() <= 1e-9
        if st1 == capi.LL_OK and r1.registered:
            p = oracle.default_params(q_w_last=q, t_w_last=tt, q_w_curr=q, t_w_curr=tt)
            ost, ores = oracle.register(g["map_corner"], trees[0], g["map_surf"], trees[1], fc, fs, p)
            assert r.status == ost and np.linalg.norm(np.array(r.t_w_curr) - np.array(ores.t_w_curr)) < 1e-7
            assert np.abs(np.array(r.q_w_curr) - np.array(ores.q_w_curr)).max() < 1e-7   # (components: quat_angle's acos resolves nothing below ~1.5e-8)
    ok = [j for j, r in enumerate(out["refined"]) if out["item_status"][j] == 0 and r.registered == 1 and r.status == 1]
    want = min(ok, key=lambda j: (out["refined"][j].inlier_threshold, j)) if ok else -1
    assert out["best"] == want
    idx.close()


# ---------------------------------------------------------------------------------------------- end to end in the C2 room
def _c2_features(ctx, pose, n=100000, seed=S.SEED + 77):
    from loam_livox_b200.registration import Livox_laser, voxel_grid_filter
    lx = Livox_laser(ctx)
    lx.extract_laser_features(S.make_scan(n, pose, seed=seed), 100.0)
    c, s, _ = lx.get_features(0.0, 1.0)
    return voxel_grid_filter(ctx, voxel_grid_filter(ctx, c, 0.1), 0.2), voxel_grid_filter(ctx, voxel_grid_filter(ctx, s, 0.2), 0.4)


def test_end_to_end_c2_room(ctxs, c2):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import RelocIndex, relocalize, voxel_grid_filter, window_lattice, yaw_circle
    mc, ms, m = c2
    # The room repeats itself every 4 m in x (the pillar pitch) and the floor, ceiling and side walls score at any x: over the whole room the
    # refinement of an alias 8 m away registers as well as the truth (measured: DESIGN.md §4.3).  So the window spans one pitch in x around the
    # truth, the whole width in y and every yaw, and the pose is close to a hypothesis (a yaw error of a few degrees moves the far end wall out of
    # its dilated voxels).
    truth = S.Pose(S.quat_from_euler(0.0, 0.0, np.radians(0.5)), np.array([10.05, -0.97, 0.1]))
    fc, fs = _c2_features(ctxs[0], truth)
    window = ((8.0, 12.0, 1.0), ROOM[1], (truth.t[2], truth.t[2], 0.0))
    idx = RelocIndex(ctxs[0], m, 0.2, 1, 1 << 16)
    pts = voxel_grid_filter(ctxs[0], np.concatenate([fc, fs]), 0.5)
    # NumPy first: the true basin holds the top peak, uniquely
    d, lo, grid = R.index([mc, ms], 0.2, 1)[:3]
    rot = yaw_circle(10.0)
    t0, step, nt = window_lattice(window)
    sc = R.scores(grid, d, lo, 0.2, 1, pts, rot, t0, step, nt)
    hs, ss = R.peaks(sc, rot.shape[0], nt, True)
    q0, t0_ = R.candidate_pose(hs[0], rot, t0, step, nt)
    assert np.linalg.norm(t0_[:2] - truth.t[:2]) < 0.5 and np.degrees(S.quat_angle(q0, truth.q)) < 5.5 and ss[1] < ss[0]
    out = relocalize(ctxs[0], m, idx, fc, fs, window=window, yaw_step_deg=10.0, k=8, score_pts=pts)
    assert out["candidates"][0]["hypothesis"] == hs[0]
    b = out["best"]
    assert b >= 0
    r = out["refined"][b]
    assert np.linalg.norm(np.array(r.t_w_curr) - truth.t) < 0.05 and np.degrees(S.quat_angle(np.array(r.q_w_curr), truth.q)) < 0.5
    # every candidate rejected by the final-cost gate (:561-573): best = -1, still LL_OK
    st = capi.default_reg_state(max_final_cost=0.0)
    st.current_frame_index = st.mapping_init_accumulate_frames + 1
    out0 = relocalize(ctxs[0], m, idx, fc, fs, window=window, yaw_step_deg=10.0, k=8, score_pts=pts, state=st)
    assert out0["best"] == -1 and len(out0["refined"]) > 0 and all(x.status == 0 for x in out0["refined"])
    idx.close()


# ---------------------------------------------------------------------------------------------- validation
def _raw_call(ctx, m, idx, pts, fc, fs, cfg, st, K=16):
    from loam_livox_b200 import capi
    cand, res, status = (capi.RelocCandidate * K)(), (capi.RegResult * K)(), (C.c_int * K)()
    n, best = C.c_int(), C.c_int()
    rc = ctx._lib.ll_relocalize(ctx.h, m.h if m else None, idx.h if idx else None, pts.ctypes.data, pts.shape[0], fc.ctypes.data, fc.shape[0], fs.ctypes.data, fs.shape[0],
                                capi.LL_FMT_XYZI16, capi.LL_HOST, C.byref(cfg) if cfg is not None else None, C.byref(st), cand, res, status, C.byref(n), C.byref(best))
    val = lambda x: np.array(list(x) if isinstance(x, C.Array) else [x]).tobytes()  # noqa: E731
    key = [tuple(val(getattr(cand[i], f)) for f, _ in capi.RelocCandidate._fields_) + tuple(val(getattr(res[i], f)) for f, _ in capi.RegResult._fields_ if not f.startswith("gpu_ms"))
           + (status[i],) for i in range(n.value)]
    return rc, key, best.value


def test_validation_leaves_the_context_usable(ctxs):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Context, Map, RelocIndex, reloc_cfg, yaw_circle
    ctx = ctxs[0]
    g, m, idx, pts = _golden_case(ctx)
    fc, fs = np.ascontiguousarray(g["feat_corner"], np.float32), np.ascontiguousarray(g["feat_surf"], np.float32)
    t = g["guess_t"]
    rot = yaw_circle(30.0)
    good, _k1 = reloc_cfg(rot, (t[0] - 0.3, t[1] - 0.3, t[2]), (0.3, 0.3, 1.0), (3, 3, 1), k=4)
    st = capi.default_reg_state(current_frame_index=51, mapping_init_accumulate_frames=50)
    L = ctx._lib
    # the index build
    h = C.c_void_p()
    for res, dil, mh, code in ((0.0, 1, 10, capi.LL_ERR_INVALID), (-1.0, 1, 10, capi.LL_ERR_INVALID), (0.3, 5, 10, capi.LL_ERR_INVALID), (0.3, -1, 10, capi.LL_ERR_INVALID),
                               (0.3, 1, 0, capi.LL_ERR_INVALID), (0.3, 1, (1 << 24) + 1, capi.LL_ERR_INVALID), (1e-4, 1, 10, capi.LL_ERR_CAPACITY)):
        assert L.ll_reloc_index_build(ctx.h, m.h, res, dil, mh, C.byref(h)) == code, (res, dil, mh)
    sharded = Map(ctx, g["map_corner"], g["map_surf"], rank=0, world=2)
    assert L.ll_reloc_index_build(ctx.h, sharded.h, 0.3, 1, 10, C.byref(h)) == capi.LL_ERR_INVALID
    # the relocalization
    bad_q = rot.copy(); bad_q[1] *= 1.001
    cfgs = {
        "non-unit": (reloc_cfg(bad_q, good.t0, good.step, good.nt, 4), capi.LL_ERR_INVALID),
        "nt 0": (reloc_cfg(rot, good.t0, good.step, (3, 0, 1), 4), capi.LL_ERR_INVALID),
        "n_rot 0": (reloc_cfg(rot[:0], good.t0, good.step, good.nt, 4), capi.LL_ERR_INVALID),
        "hypotheses": (reloc_cfg(rot, good.t0, good.step, (20, 20, 1), 4), capi.LL_ERR_INVALID),   # 12 x 400 > 4096
        "K 0": (reloc_cfg(rot, good.t0, good.step, good.nt, 0), capi.LL_ERR_INVALID),
        "K 17": (reloc_cfg(rot, good.t0, good.step, good.nt, 17), capi.LL_ERR_INVALID),
    }
    for name, ((cfg, _keep), code) in cfgs.items():
        assert _raw_call(ctx, m, idx, pts, fc, fs, cfg, st)[0] == code, name
    assert _raw_call(ctx, m, idx, pts, fc, fs, None, st)[0] == capi.LL_ERR_INVALID
    gated = capi.default_reg_state(current_frame_index=50, mapping_init_accumulate_frames=50)
    assert _raw_call(ctx, m, idx, pts, fc, fs, good, gated)[0] == capi.LL_ERR_INVALID
    other = Map(ctx, g["map_corner"], g["map_surf"])
    assert _raw_call(ctx, other, idx, pts, fc, fs, good, st)[0] == capi.LL_ERR_INVALID
    assert _raw_call(ctx, sharded, idx, pts, fc, fs, good, st)[0] == capi.LL_ERR_INVALID
    many = np.zeros((capi.LL_RELOC_MAX_SCORE_POINTS + 1, 4), np.float32)
    assert _raw_call(ctx, m, idx, many, fc, fs, good, st)[0] == capi.LL_ERR_CAPACITY
    big_fc = np.ascontiguousarray(np.tile(fc, (200, 1)))
    big_fs = np.ascontiguousarray(np.tile(fs, (200, 1)))
    assert 4 * (big_fc.shape[0] + big_fs.shape[0]) > ctx.cfg.max_features
    assert _raw_call(ctx, m, idx, pts, big_fc, big_fs, good, st)[0] == capi.LL_ERR_CAPACITY
    # usable afterwards: the next call is a fresh context's
    rc, key, best = _raw_call(ctx, m, idx, pts, fc, fs, good, st)
    fresh = Context(0, max_scan_points=200000, max_features=400000)
    rc2, key2, best2 = _raw_call(fresh, m, idx, pts, fc, fs, good, st)
    assert rc == rc2 == capi.LL_OK and key == key2 and best == best2 and len(key) > 0
    fresh.close(); idx.close()


# ---------------------------------------------------------------------------------------------- the streaming mapper
N = 24000


def _mapper(ctx, mode, init=3, window=400, **reg):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping
    pipe = capi.PipelineCfg(pieces=3, use_piece=0, extractor_leaf_corner=0.1, extractor_leaf_surf=0.2, mapping_leaf_corner=0.1, mapping_leaf_surf=0.4, whole_frame=1)
    return Laser_mapping(ctx, reg=capi.default_reg_state(mapping_init_accumulate_frames=init, **reg), pipeline=pipe, matching_mode=mode, maximum_history_size=window)


def _stream(n, seed=S.SEED + 500, n_points=N):
    poses = S.trajectory(n_scans=n, n_static=4, speed=1.0)
    return poses, [S.make_scan(n_points, p, seed=seed + k) for k, p in enumerate(poses)], [100.0 + 0.1 * k for k in range(n)]


def _entry(res):
    from loam_livox_b200 import capi
    return tuple(np.array(list(getattr(res, f)) if isinstance(getattr(res, f), C.Array) else [getattr(res, f)]).tobytes()
                 for f, _ in capi.RegResult._fields_ if not f.startswith("gpu_ms"))


def _section(img, k):
    off, length = struct.unpack_from("<QQ", img, 24 + 16 * k)
    return img[off:off + length]


@pytest.mark.parametrize("mode", [0, 1])
def test_whole_map_equals_a_build_from_the_image(ctxs, mode):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Map, voxel_grid_filter
    ctx = ctxs[0]
    _, raws, stamps = _stream(9)
    gm = _mapper(ctx, mode, window=4)
    for k in range(9):
        gm.process_new_scan(raws[k], stamps[k])
    img = gm.save()
    wm = gm.whole_map()
    assert gm.save() == img   # the mapper is not modified
    clouds = []
    for c in range(2):
        if mode == 0:
            h = _section(img, capi.LL_IMAGE_HISTORY_CORNER + c)
            ns, npts = struct.unpack_from("<qq", h, 0)
            p = np.frombuffer(h, np.float32, count=4 * npts, offset=16 + 4 * ns).reshape(-1, 4)
        else:
            h = _section(img, capi.LL_IMAGE_CELLS_CORNER + c)
            _, _, ncell, npts = struct.unpack_from("<iiqq", h, 0)
            p = np.frombuffer(h, np.float32, count=4 * npts, offset=24 + 16 * ncell).reshape(-1, 4).copy()
            p[:, 3] = 0.0
        clouds.append(voxel_grid_filter(ctx, p, (0.1, 0.4)[c]))
    ref = Map(ctx, clouds[0], clouds[1])
    rng = np.random.default_rng(mode)
    q = np.concatenate([clouds[1][rng.integers(0, clouds[1].shape[0], 3000), :3] + rng.normal(0, 0.3, (3000, 3)).astype(np.float32),
                        np.zeros((3000, 1), np.float32)], axis=1).astype(np.float32)
    for which in (0, 1):
        assert wm.size(which) == ref.size(which) == clouds[which].shape[0]
        i1, d1 = wm.nearestKSearch(which, q)
        i2, d2 = ref.nearestKSearch(which, q)
        assert np.array_equal(i1, i2) and np.array_equal(d1, d2)
    gm.close()


@pytest.mark.parametrize("mode,reject", [(0, False), (1, False), (1, True)])
def test_set_pose_to_its_own_pose_changes_nothing(ctxs, mode, reject):
    a_ctx, b_ctx = ctxs
    _, raws, stamps = _stream(12, seed=S.SEED + 900)
    reg = dict(para_max_angular_rate=1e-9) if reject else {}   # every registered scan rejected: the match map stays as the last refresh left it
    a, b = _mapper(a_ctx, mode, **reg), _mapper(b_ctx, mode, **reg)
    for k in range(7):
        ra, _ = a.process_new_scan(raws[k], stamps[k])
        b.process_new_scan(raws[k], stamps[k])
    if reject:
        assert ra.registered == 1 and ra.status == 0
    q, t, _ = b.pose()
    b.set_pose(q.copy(), t.copy())
    for k in range(7, 12):
        ra, _ = a.process_new_scan(raws[k], stamps[k])
        rb, _ = b.process_new_scan(raws[k], stamps[k])
        assert _entry(ra) == _entry(rb), k
        b.set_pose(*b.pose()[:2])
    qa, ta, fa = a.pose()
    qb, tb, fb = b.pose()
    assert qa.tobytes() == qb.tobytes() and ta.tobytes() == tb.tobytes() and fa == fb
    a.close(); b.close()


@pytest.mark.parametrize("mode", [0, 1])
def test_session_restart_relocalizes_a_saved_mapper(ctxs, mode):
    """Save at scan k0, load on a fresh context, relocalize scan k0 + 20 without a guess, set the pose and go on for 10 scans: every scan accepted,
    and every pose within 0.05 m / 0.5 deg of the synthetic truth beyond the error of the mapper that ran the whole stream at that scan (this
    stream's odometry itself drifts about 0.1 m in y from the truth, so the restart is held to the stream's own tracking, not to zero)."""
    from loam_livox_b200.registration import Context, Laser_mapping, Livox_laser, RelocIndex, relocalize, voxel_grid_filter
    k0 = 12
    poses, raws, stamps = _stream(k0 + 31, seed=S.SEED + 1300)
    p0 = poses[0]   # the mapper's world frame is the synthetic one
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
    idx = RelocIndex(ctx, m, 0.2, 1, 1 << 16)
    k = k0 + 20
    lx = Livox_laser(ctx)
    lx.extract_laser_features(raws[k], stamps[k])
    c, s, _ = lx.get_features(0.0, 1.0)
    fc = voxel_grid_filter(ctx, voxel_grid_filter(ctx, c, 0.1), 0.1)
    fs = voxel_grid_filter(ctx, voxel_grid_filter(ctx, s, 0.2), 0.4)
    out = relocalize(ctx, m, idx, fc, fs, score_leaf=0.3, window=((-1.0, 3.0, 0.5), (-2.0, 2.0, 0.5), (poses[k].t[2], poses[k].t[2], 0.0)), yaw_step_deg=10.0, k=8)
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
    idx.close(); m.release(); lm.close(); ctx.close()
