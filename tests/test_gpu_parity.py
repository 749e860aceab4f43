"""GPU parity tests: the CUDA path (through the C-ABI) against the CPU oracle on identical seeded inputs.

Bars: bit-exact for integer / index / fp32 work (masks, labels, voxel centroids, neighbour ids and fp32 squared
distances); fp64 solver quantities to 1e-9 relative; final pose within north_star's 1e-4 m / 1e-4 rad.
"""
import numpy as np
import pytest

from loam_livox_b200 import synthetic as S

pytestmark = pytest.mark.gpu


def _mk(nc, ns, qc, qs, seed=0):
    mc, ms = S.make_map(nc, ns, seed=S.SEED + seed)
    pose = S.default_pose()
    fc, fs = S.make_features(qc, qs, pose, seed=S.SEED + seed)
    return mc, ms, fc, fs, pose


# ---------------------------------------------------------------------------------------------- K5/K6 kNN
@pytest.mark.parametrize("n_map,nq", [(40, 64), (1000, 500), (45000, 4000), (300000, 20000)])
def test_knn_bit_exact(ctx, oracle, n_map, nq):
    from loam_livox_b200.registration import Map
    mc, ms = S.make_map(max(n_map // 9, 8), n_map)
    rng = np.random.default_rng(n_map)
    q = ms[rng.integers(0, ms.shape[0], nq)].copy()
    q[:, :3] += rng.normal(0, 0.05, (nq, 3)).astype(np.float32)
    m = Map(ctx, mc, ms)
    idx, d2 = m.nearestKSearch(1, q)
    tree = oracle.KdTree(ms)
    oi, od, _ = tree.knn(q)
    assert np.array_equal(d2, od), "fp32 squared distances must be bit-exact (FLANN L2_Simple order)"
    assert np.array_equal(idx, oi)
    idxc, d2c = m.nearestKSearch(0, q[: min(nq, 200)])
    bi, bd, _ = oracle.knn_brute(mc, q[: min(nq, 200)])
    assert np.array_equal(d2c, bd) and np.array_equal(idxc, bi)


def test_knn_edge_cases(ctx, oracle):
    from loam_livox_b200.registration import Map
    rng = np.random.default_rng(5)
    # fewer than 5 points, duplicates (ties), NaN points in the map, far-away queries
    ms = rng.normal(0, 1, (3, 4)).astype(np.float32)
    mc = np.concatenate([rng.normal(0, 1, (50, 4)), np.full((3, 4), np.nan)]).astype(np.float32)
    mc[10:20] = mc[0]   # exact duplicates -> ties broken by index
    m = Map(ctx, mc, ms)
    q = rng.normal(0, 3, (100, 4)).astype(np.float32)
    idx, d2 = m.nearestKSearch(1, q)
    bi, bd, _ = oracle.knn_brute(ms, q)
    assert np.array_equal(idx, bi) and np.array_equal(d2, bd)
    assert (idx[:, 3:] == -1).all() and np.isinf(d2[:, 3:]).all()
    idx, d2 = m.nearestKSearch(0, q)
    bi, bd, _ = oracle.knn_brute(mc, q)
    assert np.array_equal(idx, bi) and np.array_equal(d2, bd)


# ---------------------------------------------------------------------------------------------- K4 VoxelGrid
@pytest.mark.parametrize("n,leaf", [(1, 0.4), (1000, 0.1), (50000, 0.4), (200000, 0.05)])
def test_voxel_grid_bit_exact(ctx, oracle, n, leaf):
    from loam_livox_b200.registration import voxel_grid_filter
    _, ms = S.make_map(8, n, seed=n)
    ms[:, 3] = np.random.default_rng(n).uniform(0, 0.1, n)
    if n > 10:
        ms[3, 0] = np.nan
    out = voxel_grid_filter(ctx, ms, leaf)
    ref = oracle.voxel_grid(ms, leaf)
    assert out.shape == ref.shape
    assert np.array_equal(out, ref)


def test_voxel_grid_overflow_passthrough(ctx, oracle):
    from loam_livox_b200.registration import voxel_grid_filter
    rng = np.random.default_rng(3)
    p = rng.uniform(-1000, 1000, (500, 4)).astype(np.float32)
    out = voxel_grid_filter(ctx, p, 0.001)   # (2e6)^3 voxels overflow int32 -> PCL passes the input through
    assert np.array_equal(out, oracle.voxel_grid(p, 0.001)) and out.shape[0] == 500


# ---------------------------------------------------------------------------------------------- K1-K3 extractor
@pytest.mark.parametrize("n", [10000, 100000])
def test_extractor_bit_exact(ctx, oracle, n):
    from loam_livox_b200.registration import Livox_laser
    sc = S.make_scan(n)
    sc[50:53, :3] = 0.0          # a run of zero returns
    sc[200, :3] = np.nan
    sc[201, :3] = 0.0            # zero return right after a NaN
    ex = oracle.Extractor()
    gl = Livox_laser(ctx)
    for k, stamp in enumerate((100.0, 100.1)):   # two frames: exercises the timestamp bookkeeping
        ns_o = ex.extract(sc, stamp)
        ns_g = gl.extract_laser_features(sc, stamp)
        assert ns_g == ns_o
        io, ig = ex.point_info(), gl.point_info()
        for key in ("pt_type", "pt_label", "polar_direction"):
            assert np.array_equal(io[key], ig[key]), key
        for key in ("curvature", "view_angle", "depth_sq2", "time_stamp", "polar_dis_sq2"):
            assert np.array_equal(io[key], ig[key], equal_nan=True), key
        assert np.array_equal(ex.split_idx(), gl.split_idx())
        so, eo = ex.piece_bounds(3)
        sg, eg = gl.piece_bounds(3)
        assert np.array_equal(so, sg) and np.array_equal(eo, eg)
        for (a, b) in ((0.0, 1.0), (float(so[1]), float(eo[1]))):
            co, su, fu = ex.get_features(a, b)
            cg, sg2, fg = gl.get_features(a, b)
            assert np.array_equal(co, cg) and np.array_equal(su, sg2) and np.array_equal(fu, fg, equal_nan=True)
            assert co.shape[0] > 0 and su.shape[0] > 100


# ---------------------------------------------------------------------------------------------- K6-K10 pieces
def test_blocks_normal_equations_and_solve(ctx, oracle):
    from loam_livox_b200.registration import Map, Point_cloud_registration
    mc, ms, fc, fs, pose = _mk(5000, 45000, 1000, 9000)
    guess = S.perturb_pose(pose, np.random.default_rng(1))
    m = Map(ctx, mc, ms)
    reg = Point_cloud_registration(ctx)
    reg.set_pose(guess.q, guess.t)
    typ, a3, v3, ca, sa = reg.build_blocks(m, fc, fs)
    tc, ts = oracle.KdTree(mc), oracle.KdTree(ms)
    p = oracle.default_params(q_w_last=guess.q, t_w_last=guess.t, q_w_curr=guess.q, t_w_curr=guess.t)
    blocks, src, oca, osa = oracle.build_blocks(mc, tc, ms, ts, fc, fs, p)
    assert (ca, sa) == (oca, osa)
    slot = src[:, 1] + np.where(src[:, 0] == 1, fc.shape[0], 0)
    assert np.array_equal(np.nonzero(typ)[0], slot)
    assert np.array_equal(typ[slot], blocks[:, 0].astype(np.int32) + 1)
    assert np.array_equal(a3[slot], blocks[:, 4:7])
    assert np.allclose(v3[slot], blocks[:, 7:10], rtol=0, atol=1e-15)
    # normal equations at a non-trivial x
    d = np.array([0.01, -0.02, 0.015, 0.05, -0.04, 0.03])
    x = oracle.plus([0, 0, 0, 1, 0, 0, 0], d)
    H, g, cost = reg.normal_equations(x)
    oc, og, oH = oracle.evaluate(blocks, guess.q, guess.t, x)
    assert abs(cost - oc) <= 1e-10 * abs(oc)
    assert np.allclose(g, og, rtol=1e-9, atol=1e-9 * np.abs(og).max())
    assert np.allclose(H, oH, rtol=1e-9, atol=1e-9 * np.abs(oH).max())
    # one ceres::Solve-equivalent
    for iters in (2, 50):
        xg, ic, fcst, it = reg.solve([0, 0, 0, 1, 0, 0, 0], iters)
        xo, so = oracle.solve(blocks, guess.q, guess.t, [0, 0, 0, 1, 0, 0, 0], iters)
        assert it == int(so["iterations"])
        assert abs(ic - so["initial_cost"]) <= 1e-10 * so["initial_cost"] and abs(fcst - so["final_cost"]) <= 1e-9 * so["final_cost"]
        assert np.allclose(xg, xo, rtol=0, atol=1e-9)


@pytest.mark.parametrize("cfg", [(5000, 45000, 1000, 9000), (20000, 180000, 3000, 27000),
                                 (20000, 180000, 4000, 36000), (50000, 450000, 15000, 135000)])   # 40k / 150k features: 2 and 5 tiles per solver CTA
def test_register_pose_parity(ctx, oracle, cfg):
    from loam_livox_b200.registration import Map, Point_cloud_registration
    mc, ms, fc, fs, pose = _mk(*cfg)
    m = Map(ctx, mc, ms)
    tc, ts = oracle.KdTree(mc), oracle.KdTree(ms)
    for seed in range(3 if cfg[2] + cfg[3] <= 30000 else 1):   # one start point at the multi-tile sizes (the oracle's CPU time)
        guess = S.perturb_pose(pose, np.random.default_rng(seed))
        reg = Point_cloud_registration(ctx)
        reg.set_pose(guess.q, guess.t)
        st = reg.find_out_incremental_transfrom(m, fc, fs)
        p = oracle.default_params(q_w_last=guess.q, t_w_last=guess.t, q_w_curr=guess.q, t_w_curr=guess.t)
        ost, ores = oracle.register(mc, tc, ms, ts, fc, fs, p)
        r = reg.result
        assert st == ost == 1 and r.registered == 1
        assert r.icp_iterations == ores.icp_iterations
        assert (r.corner_used, r.surf_used, r.num_residual_blocks) == (ores.corner_used, ores.surf_used, ores.num_residual_blocks)
        dt = np.linalg.norm(np.array(r.t_w_curr) - np.array(ores.t_w_curr))
        da = S.quat_angle(np.array(r.q_w_curr), np.array(ores.q_w_curr))
        assert dt < 1e-4 and da < 1e-4, (dt, da)          # north_star tolerance
        assert dt < 1e-7 and da < 1e-7, (dt, da)          # what we actually expect
        assert abs(r.final_cost - ores.final_cost) <= 1e-7 * ores.final_cost
        assert abs(r.inlier_threshold - ores.inlier_threshold) <= 1e-7 * ores.inlier_threshold
        # and the registration recovers the injected motion
        assert np.linalg.norm(np.array(r.t_w_curr) - pose.t) < 5e-3 and S.quat_angle(np.array(r.q_w_curr), pose.q) < 1e-3


def test_register_gate_and_reject(ctx, oracle):
    from loam_livox_b200.registration import Map, Point_cloud_registration
    mc, ms, fc, fs, pose = _mk(500, 4500, 200, 1800)
    m = Map(ctx, mc, ms)
    # first frames: returns 1 without registering (:199)
    reg = Point_cloud_registration(ctx, current_frame_index=10)
    reg.set_pose(pose.q, pose.t)
    assert reg.find_out_incremental_transfrom(m, fc, fs) == 1 and reg.result.registered == 0
    assert np.allclose(reg.m_t_w_curr, pose.t)
    # reject gate on the final cost (:561-573): pose reverted, status 0
    guess = S.perturb_pose(pose, np.random.default_rng(2))
    reg = Point_cloud_registration(ctx, max_final_cost=1e-9)
    reg.set_pose(guess.q, guess.t)
    assert reg.find_out_incremental_transfrom(m, fc, fs) == 0
    assert np.allclose(reg.m_t_w_curr, guess.t) and np.allclose(reg.m_q_w_curr, guess.q)


def test_transform_bit_exact(ctx, oracle):
    from loam_livox_b200.registration import Point_cloud_registration
    pose = S.default_pose()
    _, fs = S.make_features(10, 5000, pose)
    reg = Point_cloud_registration(ctx)
    out = reg.pointcloudAssociateToMap(fs, pose.q, pose.t)
    assert np.array_equal(out, oracle.transform(fs, pose.q, pose.t))


# ---------------------------------------------------------------------------------------------- whole per-scan step
def test_scan_to_pose_matches_staged_oracle(ctx, oracle):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Map, scan_to_pose
    pose = S.default_pose()
    mc, ms = S.make_map(20000, 200000)
    raw = S.make_scan(20000, pose)
    m = Map(ctx, mc, ms)
    guess = S.perturb_pose(pose, np.random.default_rng(4), dt=0.05, dang_deg=1.0)
    pc = capi.PipelineCfg(pieces=3, use_piece=0, extractor_leaf_corner=0.1, extractor_leaf_surf=0.2, mapping_leaf_corner=0.1, mapping_leaf_surf=0.4, whole_frame=1)
    st = capi.default_reg_state(q_w_last=guess.q, t_w_last=guess.t, q_w_curr=guess.q, t_w_curr=guess.t)
    res, nc, ns = scan_to_pose(ctx, m, raw, 100.0, pc, st)
    # oracle, stage by stage
    ex = oracle.Extractor()
    ex.extract(raw, 100.0)
    c, s, _ = ex.get_features(0.0, 1.0)
    c = oracle.voxel_grid(oracle.voxel_grid(c, 0.1), 0.1)
    s = oracle.voxel_grid(oracle.voxel_grid(s, 0.2), 0.4)
    assert (nc, ns) == (c.shape[0], s.shape[0])
    p = oracle.default_params(q_w_last=guess.q, t_w_last=guess.t, q_w_curr=guess.q, t_w_curr=guess.t)
    ost, ores = oracle.register(mc, oracle.KdTree(mc), ms, oracle.KdTree(ms), c, s, p)
    assert res.status == ost and res.icp_iterations == ores.icp_iterations
    assert np.linalg.norm(np.array(res.t_w_curr) - np.array(ores.t_w_curr)) < 1e-6
    assert S.quat_angle(np.array(res.q_w_curr), np.array(ores.q_w_curr)) < 1e-6


# ---------------------------------------------------------------------------------------------- committed golden vectors
def test_gpu_matches_golden_file(ctx):
    """The CUDA path against tests/golden/golden_small.npz (made by tests/golden/make_golden.py from the oracle)."""
    import os
    from loam_livox_b200.registration import Livox_laser, Map, Point_cloud_registration, voxel_grid_filter
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "golden_small.npz"))
    gl = Livox_laser(ctx)
    assert gl.extract_laser_features(g["raw"], 100.0) == int(g["n_scans"])
    info = gl.point_info()
    for k in ("pt_type", "pt_label", "curvature", "view_angle"):
        assert np.array_equal(info[k], g[k], equal_nan=True), k
    assert np.array_equal(gl.split_idx(), g["split_idx"])
    c, s, f = gl.get_features(0.0, 1.0)
    assert np.array_equal(c, g["corners"]) and np.array_equal(s, g["surface"]) and f.shape[0] == int(g["n_full"])
    ps, pe = gl.piece_bounds(3)
    assert np.array_equal(ps, g["piece_start"]) and np.array_equal(pe, g["piece_end"])
    assert np.array_equal(voxel_grid_filter(ctx, g["map_surf"], 0.4), g["voxel"])
    m = Map(ctx, g["map_corner"], g["map_surf"])
    ki, kd = m.nearestKSearch(1, g["knn_q"])
    assert np.array_equal(ki, g["knn_idx"]) and np.array_equal(kd, g["knn_d2"])
    reg = Point_cloud_registration(ctx)
    reg.set_pose(g["guess_q"], g["guess_t"])
    typ, a3, v3, ca, sa = reg.build_blocks(m, g["feat_corner"], g["feat_surf"])
    assert (ca, sa, int((typ != 0).sum())) == (int(g["corner_avail"]), int(g["surf_avail"]), int(g["n_blocks"]))
    H, gr, cost = reg.normal_equations(g["eval_x"])
    assert abs(cost - float(g["eval_cost"])) <= 1e-10 * float(g["eval_cost"]) and np.allclose(H, g["eval_H"], rtol=1e-9, atol=1e-9 * np.abs(g["eval_H"]).max())
    assert np.allclose(gr, g["eval_g"], rtol=1e-9, atol=1e-9 * np.abs(g["eval_g"]).max())
    st = reg.find_out_incremental_transfrom(m, g["feat_corner"], g["feat_surf"])
    r = reg.result
    assert st == int(g["reg_status"]) and r.icp_iterations == int(g["reg_iters"]) and r.num_residual_blocks == int(g["reg_blocks"])
    assert np.linalg.norm(np.array(r.t_w_curr) - g["reg_t"]) < 1e-7 and S.quat_angle(np.array(r.q_w_curr), g["reg_q"]) < 1e-7
    assert abs(r.final_cost - float(g["reg_final_cost"])) <= 1e-7 * float(g["reg_final_cost"])
    assert abs(r.inlier_threshold - float(g["reg_inlier_thr"])) <= 1e-7 * float(g["reg_inlier_thr"])


def test_register_edge_cases(ctx, oracle):
    from loam_livox_b200.registration import Map, Point_cloud_registration, LoamLivoxError
    mc, ms, fc, fs, pose = _mk(500, 4500, 200, 1800)
    m = Map(ctx, mc, ms)
    # ragged inputs: no corner features at all / a NaN corner feature / pcl::PointXYZI (32-byte) layout
    reg = Point_cloud_registration(ctx)
    reg.set_pose(pose.q, pose.t)
    assert reg.find_out_incremental_transfrom(m, np.zeros((0, 4), np.float32), fs) == 1 and reg.result.corner_used == 0
    fc2 = fc.copy(); fc2[3, 0] = np.nan
    pcl = lambda a: np.concatenate([a[:, :3], np.ones((a.shape[0], 1), np.float32), a[:, 3:4], np.zeros((a.shape[0], 3), np.float32)], axis=1)
    reg2 = Point_cloud_registration(ctx)
    reg2.set_pose(pose.q, pose.t)
    assert reg2.find_out_incremental_transfrom(m, pcl(fc2), pcl(fs)) == 1
    p = oracle.default_params(q_w_last=pose.q, t_w_last=pose.t, q_w_curr=pose.q, t_w_curr=pose.t)
    ost, ores = oracle.register(mc, oracle.KdTree(mc), ms, oracle.KdTree(ms), fc2, fs, p)
    assert reg2.result.corner_used == ores.corner_used and np.linalg.norm(np.array(reg2.result.t_w_curr) - np.array(ores.t_w_curr)) < 1e-7
    # features far from the map: every gate fails -> explicit error instead of the reference's undefined behaviour
    far = fs.copy(); far[:, :3] += 500.0
    reg3 = Point_cloud_registration(ctx)
    reg3.set_pose(pose.q, pose.t)
    with pytest.raises(LoamLivoxError):
        reg3.find_out_incremental_transfrom(m, far[:50], far)


# ---------------------------------------------------------------------------------------------- a12 (i): residual-block cap
@pytest.mark.parametrize("cap,seed", [(200, 0), (200, 7), (150, 1), (3000, 2)])
def test_residual_cap_parity(ctx, oracle, cap, seed):
    """maximum_allow_residual_block of the shipped YAMLs (200 / 150; 3000 = only the drop rule binds, not the pre-skip): the pre-skipped feature set,
    the dropped block set (same counter-based draws as the oracle), the block counts of every ICP iteration and the pose."""
    from loam_livox_b200.registration import Map, Point_cloud_registration
    mc, ms, fc, fs, pose = _mk(5000, 45000, 1000, 9000)
    m = Map(ctx, mc, ms)
    tc, ts = oracle.KdTree(mc), oracle.KdTree(ms)
    guess = S.perturb_pose(pose, np.random.default_rng(seed))
    kw = dict(maximum_allow_residual_block=cap, rng_seed=seed)
    p = oracle.default_params(q_w_last=guess.q, t_w_last=guess.t, q_w_curr=guess.q, t_w_curr=guess.t, **kw)
    # pre-skip (:232-238, :339-345): the features that reach the kNN search in ICP iteration 0
    reg = Point_cloud_registration(ctx, **kw)
    reg.set_pose(guess.q, guess.t)
    typ, a3, v3, ca, sa = reg.build_blocks(m, fc, fs)
    blocks, src, oca, osa = oracle.build_blocks(mc, tc, ms, ts, fc, fs, p)
    slot = src[:, 1] + np.where(src[:, 0] == 1, fc.shape[0], 0)
    assert (ca, sa) == (oca, osa) and np.array_equal(np.nonzero(typ)[0], slot)
    if fs.shape[0] > 2 * cap:
        assert 0.7 * 2 * cap < sa < 1.3 * 2 * cap      # keep probability 2 cap / N
    # whole registration: same block counts after the drop (:434-458) and after the inlier selection, same pose
    st = reg.find_out_incremental_transfrom(m, fc, fs)
    ost, ores, tr = oracle.register(mc, tc, ms, ts, fc, fs, p, want_trace=True)
    r = reg.result
    assert st == ost == 1 and r.icp_iterations == ores.icp_iterations
    assert (r.corner_used, r.surf_used, r.num_residual_blocks) == (ores.corner_used, ores.surf_used, ores.num_residual_blocks)
    assert all(t.blocks_before_select <= 1.3 * cap for t in tr)
    dt = np.linalg.norm(np.array(r.t_w_curr) - np.array(ores.t_w_curr))
    da = S.quat_angle(np.array(r.q_w_curr), np.array(ores.q_w_curr))
    assert dt < 1e-7 and da < 1e-7, (dt, da)
    assert abs(r.final_cost - ores.final_cost) <= 1e-7 * ores.final_cost
    # a different seed draws a different subset
    reg2 = Point_cloud_registration(ctx, maximum_allow_residual_block=cap, rng_seed=seed + 1)
    reg2.set_pose(guess.q, guess.t)
    typ2 = reg2.build_blocks(m, fc, fs)[0]
    assert (fc.shape[0] <= 2 * cap and fs.shape[0] <= 2 * cap) or not np.array_equal(typ2 != 0, typ != 0)


def test_shipped_yaml_values_run(ctx, oracle):
    """ll_reg_state_yaml: cap 200 / 150 and max_allow_final_cost 2.0 -- the library must register a real scan under the reference's own configs."""
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Map, Point_cloud_registration
    mc, ms, fc, fs, pose = _mk(5000, 45000, 1000, 9000)
    m = Map(ctx, mc, ms)
    for realtime in (False, True):
        y = capi.yaml_reg_state(realtime)
        assert (y.maximum_allow_residual_block, y.max_final_cost) == (150 if realtime else 200, 2.0)
        guess = S.perturb_pose(pose, np.random.default_rng(11))
        reg = Point_cloud_registration(ctx)
        reg.state = capi.yaml_reg_state(realtime, rng_seed=5)
        reg.set_pose(guess.q, guess.t)
        assert reg.find_out_incremental_transfrom(m, fc, fs) == 1 and reg.result.registered == 1
        assert reg.result.num_residual_blocks <= 1.3 * y.maximum_allow_residual_block
        assert np.linalg.norm(np.array(reg.result.t_w_curr) - pose.t) < 0.03


# ---------------------------------------------------------------------------------------------- a14: device cell map, streaming mapper (C3)
@pytest.mark.gpu
def test_cellmap_append_assemble_parity(ctx, oracle):
    from loam_livox_b200.registration import Points_cloud_map
    rng = np.random.default_rng(2)
    p = np.zeros((60000, 4), np.float32)
    p[:, :3] = rng.normal(0, 4, (60000, 3)).astype(np.float32)
    p[:, 3] = rng.uniform(0, 1, 60000).astype(np.float32)                  # intensity must be dropped by the cell map
    g, o = Points_cloud_map(ctx, 1.0, 2000), oracle.CellMap(1.0, 2000)
    for lo, hi in ((0, 25000), (25000, 25001), (25001, 60000)):
        g.append_cloud(p[lo:hi]); o.append_cloud(p[lo:hi])
        assert g.stats() == (o.cells(), o.points(), o.frame_idx())
    q, t = S.quat_from_euler(0.02, -0.01, 0.4), np.array([0.5, -0.2, 0.1])
    for replace in (False, True, True):
        a, fa = g.assemble(q, t, 7.0, 45.0, 0.2, replace)
        b, fb = o.assemble(q, t, 7.0, 45.0, 0.2, replace)
        assert fa == fb and a.shape == b.shape and np.array_equal(a, b)
        assert g.stats() == (o.cells(), o.points(), o.frame_idx())
    # append after a replace, other pose, other leaf
    extra = np.zeros((5000, 4), np.float32); extra[:, :3] = rng.normal(1, 3, (5000, 3)).astype(np.float32)
    g.append_cloud(extra); o.append_cloud(extra)
    q2, t2 = S.quat_from_euler(0.0, 0.1, -2.0), np.array([-1.0, 0.3, 0.0])
    a, fa = g.assemble(q2, t2, 100.0, 45.0, 0.4, True)
    b, fb = o.assemble(q2, t2, 100.0, 45.0, 0.4, True)
    assert fa == fb and np.array_equal(a, b) and g.stats() == (o.cells(), o.points(), o.frame_idx())
    # nothing in range
    a, fa = g.assemble(q2, np.array([500.0, 0, 0]), 5.0, 45.0, 0.4, True)
    assert a.shape[0] == 0 and fa == 0


@pytest.mark.gpu
def test_cellmap_revisit_parity(ctx, oracle):
    from loam_livox_b200.registration import Points_cloud_map
    rng = np.random.default_rng(3)
    g, o = Points_cloud_map(ctx, 1.0, 3), oracle.CellMap(1.0, 3)
    near = np.zeros((2000, 4), np.float32); near[:, :3] = rng.uniform(0, 3, (2000, 3)).astype(np.float32)
    far = np.zeros((2000, 4), np.float32); far[:, :3] = rng.uniform(10, 13, (2000, 3)).astype(np.float32)
    seq = [near[:1000], far[:700], far[700:1400], far[1400:], near[1000:1500], near[1500:], far[:10]]
    for c in seq:
        g.append_cloud(c); o.append_cloud(c)
        assert g.stats() == (o.cells(), o.points(), o.frame_idx())
    q, t = np.array([1.0, 0, 0, 0]), np.array([-5.0, 1.5, 1.5])
    a, fa = g.assemble(q, t, 100.0, 45.0, 0.1, False)
    b, fb = o.assemble(q, t, 100.0, 45.0, 0.1, False)
    assert fa == fb and np.array_equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,window", [(0, 400), (0, 3), (1, 400)])
def test_streaming_mapper_parity(ctx, oracle, mode, window):
    """Config C3 in small: the device mapper against the oracle's process_new_scan loop, scan by scan (pose within 1e-4 m / 1e-4 rad), in
    matching_mode 0 (history window, the shipped YAMLs' mode; window = 3 exercises the pop at :1468-1478) and 1 (cell map)."""
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping
    poses = S.trajectory(n_scans=9, n_static=4, speed=1.0)
    reg = capi.default_reg_state(mapping_init_accumulate_frames=3)
    gm = Laser_mapping(ctx, reg=reg, matching_mode=mode, maximum_history_size=window)
    om = oracle.Mapper(oracle.default_params(mapping_init_accumulate_frames=3, num_threads=4), threads=4, matching_mode=mode, maximum_history_size=window)
    for k, pose in enumerate(poses):
        raw = S.make_scan(24000, pose, seed=S.SEED + k)
        res, stats = gm.process_new_scan(raw, 100.0 + 0.1 * k)
        ost, oq, ot = om.process_scan(raw, 100.0 + 0.1 * k)
        assert res.status == ost
        assert (stats.n_corner, stats.n_surf) == (om.last["n_corner"], om.last["n_surf"])
        assert (stats.map_corner, stats.map_surf) == (om.last["map_corner"], om.last["map_surf"]), k
        assert (stats.appended_corner, stats.appended_surf) == (om.last["appended_corner"], om.last["appended_surf"]), k
        q, t, f = gm.pose()
        assert f == om.frame_index
        assert np.linalg.norm(t - ot) < 1e-4 and S.quat_angle(q, oq) < 1e-4, (k, t, ot)
        # init_pointcloud_registration copies m_current_frame_index BEFORE the increment (laser_mapping.hpp:1349-1350): with
        # mapping_init_accumulate_frames = 3 the scans with index 0..3 are inserted unregistered, index 4 is the first ICP
        assert res.registered == (1 if k > 3 else 0), k
        if om.last["res"] is not None and om.last["res"].registered:
            assert res.registered == 1 and res.icp_iterations == om.last["res"].icp_iterations
    assert gm.pose()[2] == 9


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1])
def test_streaming_mapper_with_the_shipped_init_gate(ctx, oracle, mode):
    """mapping/init_accumulate_frames = 50 as in both YAMLs: 51 stationary scans are inserted unregistered (the registration sees the frame index before
    the increment), scan 51 is the first ICP; denser leaves than the precision YAML (what bench.py --workload c3 runs).  Counts and poses against the oracle."""
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping
    poses = S.trajectory(n_scans=58, n_static=51, speed=1.0, zero_mean_yaw=True)
    pipe = capi.PipelineCfg(pieces=3, use_piece=0, extractor_leaf_corner=0.05, extractor_leaf_surf=0.05, mapping_leaf_corner=0.05, mapping_leaf_surf=0.1, whole_frame=1)
    gm = Laser_mapping(ctx, reg=capi.default_reg_state(mapping_init_accumulate_frames=50), pipeline=pipe, line_resolution=0.05, plane_resolution=0.1, matching_mode=mode)
    om = oracle.Mapper(oracle.default_params(mapping_init_accumulate_frames=50, num_threads=8), threads=8, line_resolution=0.05, plane_resolution=0.1,
                       extractor_leaf_corner=0.05, extractor_leaf_surf=0.05, matching_mode=mode)
    for k, pose in enumerate(poses):
        raw = S.make_scan(30000, pose, seed=S.SEED + 300 + k)
        res, stats = gm.process_new_scan(raw, 100.0 + 0.1 * k)
        ost, oq, ot = om.process_scan(raw, 100.0 + 0.1 * k)
        assert res.status == ost and res.registered == (1 if k > 50 else 0), k
        assert (stats.n_corner, stats.n_surf) == (om.last["n_corner"], om.last["n_surf"]) and stats.n_surf > 1000, k
        assert (stats.map_corner, stats.map_surf) == (om.last["map_corner"], om.last["map_surf"]), k
        q, t, f = gm.pose()
        assert np.linalg.norm(t - ot) < 1e-4 and S.quat_angle(q, oq) < 1e-4, (k, t, ot)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,window", [(0, 20), (1, 400)])
def test_streaming_mapper_long_sequence(ctx, oracle, mode, window):
    """60 scans with yaw motion: the history window slides (mode 0: 20 clouds, the arenas ping-pong) / the cell maps grow and get down-sampled-and-
    replaced on every refresh (mode 1), and the two implementations must stay together (pose 1e-4, identical feature / map / append counts)."""
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping
    poses = S.trajectory(n_scans=60, n_static=4, speed=2.0, yaw_rate_deg=20.0)
    gm = Laser_mapping(ctx, reg=capi.default_reg_state(mapping_init_accumulate_frames=3), matching_mode=mode, maximum_history_size=window)
    om = oracle.Mapper(oracle.default_params(mapping_init_accumulate_frames=3, num_threads=4), threads=4, matching_mode=mode, maximum_history_size=window)
    worst = 0.0
    for k, pose in enumerate(poses):
        raw = S.make_scan(16000, pose, seed=S.SEED + 100 + k)
        res, stats = gm.process_new_scan(raw, 100.0 + 0.1 * k)
        ost, oq, ot = om.process_scan(raw, 100.0 + 0.1 * k)
        assert res.status == ost, k
        q, t, _ = gm.pose()
        worst = max(worst, float(np.linalg.norm(t - ot)), float(S.quat_angle(q, oq)))
        assert worst < 1e-4, (k, worst)
        assert (stats.map_corner, stats.map_surf, stats.appended_corner, stats.appended_surf) == \
            (om.last["map_corner"], om.last["map_surf"], om.last["appended_corner"], om.last["appended_surf"]), k
    assert gm.cfg.down_sample_replace == 1


# ---------------------------------------------------------------------------------------------- 8(e): sharded registration on >= 2 GPUs
@pytest.mark.gpu
def test_sharded_registration_two_gpus():   # halo-trimmed shards (csrc/shard.cu) + in-kernel all-reduce + L1 / count exchanges vs one GPU with the whole map
    """Spawns tests/multi_gpu/sharded_check.py under torchrun when the box has >= 2 GPUs (skipped on a one-GPU machine)."""
    import os
    import subprocess
    import sys
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", "29533",
           os.path.join(root, "tests", "multi_gpu", "sharded_check.py")]
    out = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=280)
    assert out.returncode == 0 and "SHARDED_OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]


# ---------------------------------------------------------------------------------------------- N1: motion deblur (*_mb functors)
@pytest.mark.gpu
def test_deblur_blocks_normal_equations_and_solve(ctx, oracle):
    from loam_livox_b200.registration import Map, Point_cloud_registration
    mc, ms, fc, fs, pose = _mk(5000, 45000, 1000, 9000)
    fc[:7, 3] = 0.15; fs[:9, 3] = -0.02                      # refine_blur: > 1 -> 1.0, negative stays negative
    guess = S.perturb_pose(pose, np.random.default_rng(1))
    m = Map(ctx, mc, ms)
    reg = Point_cloud_registration(ctx, if_motion_deblur=1)
    reg.set_pose(guess.q, guess.t)
    typ, a3, v3, ca, sa = reg.build_blocks(m, fc, fs)
    p = oracle.default_params(q_w_last=guess.q, t_w_last=guess.t, q_w_curr=guess.q, t_w_curr=guess.t, if_motion_deblur=1)
    blocks, src, oca, osa = oracle.build_blocks(mc, oracle.KdTree(mc), ms, oracle.KdTree(ms), fc, fs, p)
    assert (ca, sa) == (oca, osa)
    slot = src[:, 1] + np.where(src[:, 0] == 1, fc.shape[0], 0)
    assert np.array_equal(np.nonzero(typ)[0], slot) and np.array_equal(a3[slot], blocks[:, 4:7])
    for d in ([0.01, -0.02, 0.015, 0.05, -0.04, 0.03], [0, 0, 0, 0.02, 0.01, -0.03], [-0.2, 0.1, 0.05, 0.0, 0.1, 0.0]):   # slerp branch, lerp branch (w = 1), larger angle
        x = oracle.plus([0, 0, 0, 1, 0, 0, 0], d)
        H, g, cost = reg.normal_equations(x)
        oc, og, oH = oracle.evaluate(blocks, guess.q, guess.t, x)
        assert abs(cost - oc) <= 1e-10 * abs(oc)
        assert np.allclose(g, og, rtol=1e-9, atol=1e-9 * np.abs(og).max())
        assert np.allclose(H, oH, rtol=1e-9, atol=1e-9 * np.abs(oH).max())
    for iters in (2, 50):
        xg, ic, fcst, it = reg.solve([0, 0, 0, 1, 0, 0, 0], iters)
        xo, so = oracle.solve(blocks, guess.q, guess.t, [0, 0, 0, 1, 0, 0, 0], iters)
        assert it == int(so["iterations"])
        assert abs(ic - so["initial_cost"]) <= 1e-10 * so["initial_cost"] and abs(fcst - so["final_cost"]) <= 1e-9 * so["final_cost"]
        assert np.allclose(xg, xo, rtol=0, atol=1e-9)


@pytest.mark.gpu
def test_deblur_register_parity_on_distorted_scan(ctx, oracle):
    """if_motion_deblur = 1 end to end: Rodrigues-interpolated matching transform + *_mb residuals, on a scan distorted by sensor motion; at
    10 000, 40 000 and 150 000 features (1, 2 and 5 tiles per solver CTA)."""
    for nf in (10000, 40000, 150000):
        _deblur_register_parity(ctx, oracle, nf)


def _deblur_register_parity(ctx, oracle, nf):
    from loam_livox_b200.registration import Map, Point_cloud_registration
    mc, ms = S.make_map(nf // 2, 9 * nf // 2)
    m = Map(ctx, mc, ms)
    tc, ts = oracle.KdTree(mc), oracle.KdTree(ms)
    last = S.default_pose()
    motions = (((0.01, -0.02, 0.06), (0.20, -0.05, 0.02)), ((-0.03, 0.01, -0.10), (-0.10, 0.15, 0.0)))
    for k, (eul, dt) in enumerate(motions if nf == 10000 else motions[:1]):   # one motion at the multi-tile sizes (the oracle's CPU time)
        curr = S.Pose(S.quat_mul(last.q, S.quat_from_euler(*eul)), last.t + np.array(dt))
        fc, fs = S.make_distorted_features(last, curr, nf // 10, 9 * nf // 10, seed=k)
        reg = Point_cloud_registration(ctx, if_motion_deblur=1)
        reg.set_pose(last.q, last.t)
        st = reg.find_out_incremental_transfrom(m, fc, fs)
        p = oracle.default_params(q_w_last=last.q, t_w_last=last.t, q_w_curr=last.q, t_w_curr=last.t, if_motion_deblur=1)
        ost, ores = oracle.register(mc, tc, ms, ts, fc, fs, p)
        r = reg.result
        assert st == ost == 1 and r.icp_iterations == ores.icp_iterations
        assert (r.corner_used, r.surf_used, r.num_residual_blocks) == (ores.corner_used, ores.surf_used, ores.num_residual_blocks)
        dtn = np.linalg.norm(np.array(r.t_w_curr) - np.array(ores.t_w_curr)); da = S.quat_angle(np.array(r.q_w_curr), np.array(ores.q_w_curr))
        assert dtn < 1e-4 and da < 1e-4, (dtn, da)        # north_star tolerance
        assert dtn < 1e-6 and da < 1e-6, (dtn, da)
        assert abs(r.final_cost - ores.final_cost) <= 1e-6 * ores.final_cost
        assert np.linalg.norm(np.array(r.t_w_curr) - curr.t) < 0.01 and S.quat_angle(np.array(r.q_w_curr), curr.q) < 2e-3


# ---------------------------------------------------------------------------------------------- BASELINE.json full size (C2): size-independent properties
@pytest.mark.gpu
def test_full_size_map_knn_and_registration_properties(oracle):
    """100k-feature-scale queries against the 5M-point map of config C2: sampled queries agree with brute force bit for bit, every result is sorted
    and duplicate-free, re-indexing the same clouds in place changes nothing, and a registration from a perturbed pose lands on the truth."""
    from loam_livox_b200.registration import Context, Map, Point_cloud_registration
    from loam_livox_b200 import capi
    ctx = Context(0, max_scan_points=100000, max_features=100000)
    mc, ms = S.make_map(500000, 4500000)
    m = Map(ctx, mc, ms)
    assert (m.size(0), m.size(1)) == (500000, 4500000)
    pose = S.default_pose()
    fc, fs = S.make_features(3000, 60000, pose)
    world = np.concatenate([fs[:, :3] @ pose.R().T + pose.t, np.zeros((fs.shape[0], 1))], axis=1).astype(np.float32)
    idx, d2 = m.nearestKSearch(1, world)
    assert np.all(np.diff(d2, axis=1) >= 0) and np.all(idx >= 0) and np.all(idx < 4500000)
    assert all(len(set(r)) == 5 for r in idx[::97])
    sample = np.random.default_rng(5).choice(world.shape[0], 192, replace=False)
    bidx, bd2, found = oracle.knn_brute(ms, world[sample])
    assert np.array_equal(idx[sample], bidx) and np.array_equal(d2[sample], bd2)
    # in-place re-index of the same clouds: identical answers (ll_map_rebuild reuses the buffers)
    ctx.check(ctx._lib.ll_map_rebuild(ctx.h, m.h, mc.ctypes.data, mc.shape[0], ms.ctypes.data, ms.shape[0], capi.LL_FMT_XYZI16, capi.LL_HOST))
    idx2, d22 = m.nearestKSearch(1, world[:5000])
    assert np.array_equal(idx2, idx[:5000]) and np.array_equal(d22, d2[:5000])
    # registration at full feature count recovers the injected motion; running it twice gives the same bits (no order-dependent reduction)
    guess = S.perturb_pose(pose, np.random.default_rng(9))
    out = []
    for _ in range(2):
        reg = Point_cloud_registration(ctx)
        reg.set_pose(guess.q, guess.t)
        assert reg.find_out_incremental_transfrom(m, fc, fs) == 1
        out.append((np.array(reg.result.q_w_curr), np.array(reg.result.t_w_curr), reg.result.final_cost))
    assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1]) and out[0][2] == out[1][2]
    assert np.linalg.norm(out[0][1] - pose.t) < 5e-3 and S.quat_angle(out[0][0], pose.q) < 1e-3
    ctx.close()


@pytest.mark.gpu
def test_full_size_c2_pose_parity_with_the_oracle(oracle):
    """BASELINE config C2 at full size (100k-pt raw scans, 0.5M + 4.5M-pt map, the bench's pipeline leaves): two scans through ll_scan_to_pose AND
    through the oracle -- same feature counts after the four VoxelGrids, same ICP iteration count, same block counts, pose within 1e-7 (bar 1e-4)."""
    import bench
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Context, Map, scan_to_pose
    ctx = Context(0, max_scan_points=bench.N_SCAN, max_features=bench.N_SCAN)
    inputs = bench.make_inputs(0, "c2")
    mc, ms, scans, guesses, truths = inputs
    m = Map(ctx, mc, ms)
    trees = (oracle.KdTree(mc), oracle.KdTree(ms))
    ex = oracle.Extractor()
    pc = capi.PipelineCfg(**bench.PIPE)
    for k in (0, 3):
        st = capi.default_reg_state(q_w_last=guesses[k].q, t_w_last=guesses[k].t, q_w_curr=guesses[k].q, t_w_curr=guesses[k].t)
        res, nc, ns = scan_to_pose(ctx, m, scans[k], 100.0, pc, st)
        ost, ores, onc, ons = bench.oracle_step(oracle, ex, trees, mc, ms, scans[k], guesses[k], 8)
        assert (nc, ns) == (onc, ons) and ns > 20000
        assert res.status == ost == 1 and res.icp_iterations == ores.icp_iterations
        assert (res.corner_used, res.surf_used, res.num_residual_blocks) == (ores.corner_used, ores.surf_used, ores.num_residual_blocks)
        dt = np.linalg.norm(np.array(res.t_w_curr) - np.array(ores.t_w_curr))
        da = S.quat_angle(np.array(res.q_w_curr), np.array(ores.q_w_curr))
        assert dt < 1e-7 and da < 1e-7, (k, dt, da)
        assert abs(res.final_cost - ores.final_cost) <= 1e-7 * ores.final_cost
    m.release()
    ctx.close()


@pytest.mark.gpu
def test_two_contexts_on_two_host_threads_share_one_map(oracle):
    """S3 is called from up to maximum_parallel_thread std::async workers, each with its own Point_cloud_registration, sharing the read-only map
    snapshot (loam_livox/source/laser_mapping.hpp:1348,1737-1742).  Two ll_ctx on two threads against ONE ll_map: every result equals the
    result of the same registration run alone, bit for bit."""
    import threading
    from loam_livox_b200.registration import Context, Map, Point_cloud_registration
    mc, ms, fc, fs, pose = _mk(20000, 180000, 3000, 27000)
    ctxs = [Context(0, max_scan_points=40000, max_features=40000) for _ in range(2)]
    m = Map(ctxs[0], mc, ms)
    guesses = [S.perturb_pose(pose, np.random.default_rng(100 + k)) for k in range(6)]

    def run(c, g):
        reg = Point_cloud_registration(c)
        reg.set_pose(g.q, g.t)
        assert reg.find_out_incremental_transfrom(m, fc, fs) == 1
        r = reg.result
        return (tuple(r.q_w_curr), tuple(r.t_w_curr), r.final_cost, r.icp_iterations, r.num_residual_blocks)
    alone = [run(ctxs[0], g) for g in guesses]
    out = [[None] * len(guesses) for _ in range(2)]
    errs = []

    def worker(w):
        try:
            for rep in range(3):
                order = range(len(guesses)) if w == 0 else reversed(range(len(guesses)))
                for k in order:
                    out[w][k] = run(ctxs[w], guesses[k])
        except Exception as e:   # noqa: BLE001
            errs.append(e)
    ths = [threading.Thread(target=worker, args=(w,)) for w in range(2)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    assert not errs, errs
    assert out[0] == alone and out[1] == alone
    m.release()
    for c in ctxs:
        c.close()


@pytest.mark.gpu
def test_scene_alignment_parity(ctx, oracle):
    """N4: ll_scene_align against the oracle's restatement of Scene_alignment::find_tranfrom_of_two_mappings -- same number of scales, same ICP
    iteration / block counts at the last scale (the residual cap of 5000 binds: same counter-based draws), same transform."""
    from test_oracle import _two_keyframes
    from loam_livox_b200.registration import Scene_alignment
    al, ap, bl, bp, q, t = _two_keyframes()
    sa = Scene_alignment(ctx, rng_seed=4)
    r = sa.find_tranfrom_of_two_mappings(al, ap, bl, bp)
    ores, oruns = oracle.scene_align(al, ap, bl, bp, rng_seed=4, threads=8)
    assert sa.scales_run == oruns == 3
    assert (r.status, r.registered, r.icp_iterations, r.corner_used, r.surf_used, r.num_residual_blocks) == \
           (ores.status, ores.registered, ores.icp_iterations, ores.corner_used, ores.surf_used, ores.num_residual_blocks)
    dt = np.linalg.norm(np.array(r.t_w_curr) - np.array(ores.t_w_curr))
    da = S.quat_angle(np.array(r.q_w_curr), np.array(ores.q_w_curr))
    assert dt < 1e-6 and da < 1e-6, (dt, da)
    assert abs(r.inlier_threshold - ores.inlier_threshold) <= 1e-6 * abs(ores.inlier_threshold)
    assert np.linalg.norm(np.array(r.t_w_curr) - t) < 0.05 and S.quat_angle(np.array(r.q_w_curr), q) < 0.01


# ---------------------------------------------------------------------------------------------- N3: PointCloud2 payload in
@pytest.mark.gpu
def test_pointcloud2_payload_equals_float4_input(ctx, oracle):
    """A livox_ros_driver-style PointCloud2 record (x, y, z, intensity float32 + tag, line uint8; point_step 18, unaligned records) and a record with a
    uint8 intensity give exactly the features of the plain float4 input."""
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Livox_laser
    raw = S.make_scan(20000, S.default_pose())
    raw[:, 3] = np.round(np.clip(np.nan_to_num(raw[:, 3]), 0, 255))   # reflectivity as the driver sends it: integral 0..255
    gl = Livox_laser(ctx)
    n0 = gl.extract_laser_features(raw, 100.0)
    ref = gl.get_features(0.0, 1.0)
    for step, itype in ((18, capi.LL_I_FLOAT32), (13, capi.LL_I_UINT8)):
        rec = np.zeros((raw.shape[0], step), np.uint8)
        rec[:, 0:12] = raw[:, :3].copy().view(np.uint8).reshape(-1, 12)
        if itype == capi.LL_I_FLOAT32:
            rec[:, 12:16] = raw[:, 3:4].copy().view(np.uint8).reshape(-1, 4); rec[:, 16] = 7; rec[:, 17] = 3
        else:
            rec[:, 12] = raw[:, 3].astype(np.uint8)
        ctx.set_point_layout(step, 0, 4, 8, 12, itype)
        g2 = Livox_laser(ctx)
        assert g2.extract_from_pointcloud2(rec.tobytes(), raw.shape[0], 100.0) == n0
        got = g2.get_features(0.0, 1.0)
        for a, b in zip(ref, got):
            assert np.array_equal(a, b, equal_nan=True)


# ---------------------------------------------------------------------------------------------- config C5 in small: triple-lidar frame
@pytest.mark.gpu
def test_triple_lidar_frame_parity(ctx, oracle):
    """Mid-100 flow (laser_feature_extractor.hpp:303-380, launch/rosbag_mid100.launch: piecewise_number 2): ONE extractor object handles the three
    heads in turn, the per-piece feature clouds of the heads are summed, then VoxelGrid (plane_res / 2, line_res), then the registration of the merged
    300k-pt frame.  Every stage against the oracle."""
    from loam_livox_b200.registration import Livox_laser, Map, Point_cloud_registration, voxel_grid_filter
    pose = S.default_pose()
    heads = S.make_triple_scan(300000, pose)
    gl, ol = Livox_laser(ctx), oracle.Extractor()
    pieces = 2
    g_parts, o_parts = [], []
    for k, raw in enumerate(heads):
        stamp = 100.0 + 0.1 * 0 + 1e-3 * k
        ng, no = gl.extract_laser_features(raw, stamp), ol.extract(raw, stamp)
        assert ng == no and ng > 5
        gs, ge = gl.piece_bounds(pieces); os_, oe = ol.piece_bounds(pieces)
        assert np.array_equal(gs, os_) and np.array_equal(ge, oe)
        g_parts.append([gl.get_features(float(gs[i]), float(ge[i])) for i in range(pieces)])
        o_parts.append([ol.get_features(float(os_[i]), float(oe[i])) for i in range(pieces)])
    for i in range(pieces):
        gc = np.concatenate([g_parts[h][i][0] for h in range(3)]); gsf = np.concatenate([g_parts[h][i][1] for h in range(3)])
        oc = np.concatenate([o_parts[h][i][0] for h in range(3)]); osf = np.concatenate([o_parts[h][i][1] for h in range(3)])
        assert np.array_equal(gc, oc) and np.array_equal(gsf, osf)
        gsf_d, gc_d = voxel_grid_filter(ctx, gsf, 0.2), voxel_grid_filter(ctx, gc, 0.1)          # :372-373, :379-380
        assert np.array_equal(gsf_d, oracle.voxel_grid(osf, 0.2)) and np.array_equal(gc_d, oracle.voxel_grid(oc, 0.1))
        if i == 0:
            mc, ms = S.make_map(20000, 180000)
            m = Map(ctx, mc, ms)
            guess = S.perturb_pose(pose, np.random.default_rng(3), dt=0.05, dang_deg=1.0)
            fc, fs = voxel_grid_filter(ctx, gc_d, 0.1), voxel_grid_filter(ctx, gsf_d, 0.4)      # laser_mapping.hpp:1367-1373
            reg = Point_cloud_registration(ctx)
            reg.set_pose(guess.q, guess.t)
            st = reg.find_out_incremental_transfrom(m, fc, fs)
            p = oracle.default_params(q_w_last=guess.q, t_w_last=guess.t, q_w_curr=guess.q, t_w_curr=guess.t)
            ost, ores = oracle.register(mc, oracle.KdTree(mc), ms, oracle.KdTree(ms), fc, fs, p)
            assert st == ost and reg.result.icp_iterations == ores.icp_iterations
            assert np.linalg.norm(np.array(reg.result.t_w_curr) - np.array(ores.t_w_curr)) < 1e-6
            assert S.quat_angle(np.array(reg.result.q_w_curr), np.array(ores.q_w_curr)) < 1e-6


@pytest.mark.gpu
def test_frame_to_pose_equals_the_staged_triple_lidar_flow(ctx, oracle):
    """ll_frame_to_pose (three heads, one call, features never leave the device) against the oracle's staged flow: per-head extraction with ONE extractor
    object, summed feature clouds, the four VoxelGrids at the precision-YAML leaves, registration."""
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Context, Map, frame_to_pose, features_to_pointcloud2
    c3 = Context(0, max_scan_points=300000, max_features=300000)
    pose = S.default_pose()
    heads = S.make_triple_scan(300000, pose)
    stamps = [100.0 + 1e-3 * k for k in range(3)]
    mc, ms = S.make_map(20000, 180000)
    m = Map(c3, mc, ms)
    guess = S.perturb_pose(pose, np.random.default_rng(3), dt=0.05, dang_deg=1.0)
    pc = capi.PipelineCfg(pieces=2, use_piece=0, extractor_leaf_corner=0.1, extractor_leaf_surf=0.2, mapping_leaf_corner=0.1, mapping_leaf_surf=0.4, whole_frame=0)
    st = capi.default_reg_state(q_w_last=guess.q, t_w_last=guess.t, q_w_curr=guess.q, t_w_curr=guess.t)
    res, nc, ns = frame_to_pose(c3, m, heads, stamps, pc, st)
    ol = oracle.Extractor()
    oc, os_ = [], []
    for raw, stamp in zip(heads, stamps):
        assert ol.extract(raw, stamp) > 5
        a, b = ol.piece_bounds(2)
        c, s, _ = ol.get_features(float(a[0]), float(b[0]))
        oc.append(c); os_.append(s)
    fc = oracle.voxel_grid(oracle.voxel_grid(np.concatenate(oc), 0.1), 0.1)
    fs = oracle.voxel_grid(oracle.voxel_grid(np.concatenate(os_), 0.2), 0.4)
    assert (nc, ns) == (fc.shape[0], fs.shape[0])
    p = oracle.default_params(q_w_last=guess.q, t_w_last=guess.t, q_w_curr=guess.q, t_w_curr=guess.t)
    ost, ores = oracle.register(mc, oracle.KdTree(mc), ms, oracle.KdTree(ms), fc, fs, p)
    assert res.status == ost and res.icp_iterations == ores.icp_iterations
    assert np.linalg.norm(np.array(res.t_w_curr) - np.array(ores.t_w_curr)) < 1e-6 and S.quat_angle(np.array(res.q_w_curr), np.array(ores.q_w_curr)) < 1e-6
    # the output side of N3: the features as a PointCloud2 payload (x, y, z float32 at 0/4/8, intensity float32 at 16, point_step 32 -- PCL's layout)
    c3.set_point_layout(32, 0, 4, 8, 16, capi.LL_I_FLOAT32)
    for which, ref in ((0, fc), (1, fs)):
        rec = np.frombuffer(features_to_pointcloud2(c3, which), np.uint8).reshape(-1, 32)
        assert rec.shape[0] == ref.shape[0]
        xyz = rec[:, :12].copy().view(np.float32).reshape(-1, 3)
        it = rec[:, 16:20].copy().view(np.float32).reshape(-1)
        assert np.array_equal(xyz, ref[:, :3]) and np.array_equal(it, ref[:, 3]) and not rec[:, 12:16].any() and not rec[:, 20:].any()
    m.release(); c3.close()


@pytest.mark.gpu
def test_shard_build_on_one_gpu(ctx, oracle):
    """csrc/shard.cu without a second GPU: every rank's shard of a 4-way split is built on this device (ll_map_build_sharded needs no peers), and
    (1) the owner table equals the host plan, (2) the kept points are exactly the points within the halo of an owned cell (NumPy restatement), in
    input order, (3) an exact 5-NN search of a shard returns, for queries of that rank, the neighbours of the whole map whenever the 5th distance is
    inside the gate (squared distance < 50.0 / 2.0, point_cloud_registration.hpp:254,353)."""
    from test_multi_gpu_host import _numpy_shard
    from loam_livox_b200.distributed import cell_owner, plan_shards
    from loam_livox_b200.registration import Map
    mc, ms = S.make_map(3000, 60000)
    world, cell = 4, 2.0
    origin, dims, owner = plan_shards(np.concatenate([mc, ms]), world, cell)
    full = Map(ctx, mc, ms)
    rng = np.random.default_rng(8)
    q = ms[rng.integers(0, ms.shape[0], 3000)].copy(); q[:, :3] += rng.normal(0, 0.05, (3000, 3)).astype(np.float32)
    fi, fd = full.nearestKSearch(1, q)
    own_q = cell_owner(q, origin, cell, dims, owner)
    total_kept = 0
    for r in range(world):
        m = Map(ctx, mc, ms, rank=r, world=world, cell_size=cell)
        info, table = m.shard_info()
        assert np.array_equal(table, owner) and list(info.dims) == [int(v) for v in dims] and np.allclose(list(info.origin), origin)
        ks = _numpy_shard(ms, origin, cell, dims, owner, r, 50.0 ** 0.5 * 1.0001 + 1e-3)
        kc = _numpy_shard(mc, origin, cell, dims, owner, r, 2.0 ** 0.5 * 1.0001 + 1e-3)
        assert abs(int(info.kept_surf) - int(ks.sum())) <= 2 and abs(int(info.kept_corner) - int(kc.sum())) <= 2     # fp32 vs fp64 box arithmetic at the halo's rim
        assert info.kept_surf < info.total_surf == ms.shape[0]
        total_kept += int(info.kept_surf)
        sel = np.nonzero(own_q == r)[0]
        si, sd = m.nearestKSearch(1, q[sel])
        inside = fd[sel, 4] < 50.0
        assert inside.any() and np.array_equal(sd[inside], fd[sel][inside])                  # same distances ...
        kept_idx = np.nonzero(ks)[0]
        if int(info.kept_surf) == int(ks.sum()):
            assert np.array_equal(kept_idx[si[inside]], fi[sel][inside])                     # ... and the same points (shard indices -> map indices)
        m.release()
    assert total_kept > ms.shape[0]          # halos overlap: the shards together hold more than one copy
    full.release()


@pytest.mark.gpu
def test_gpu_reproduces_flann_vectors_and_cap_vectors(ctx):
    """tests/golden/golden_r2.npz: ll_knn against the answers of REAL FLANN (KDTreeSingleIndex through cv2.flann, make_golden_r2.py) on the golden map,
    and the residual cap (cap 100, seed 3) against the committed oracle vectors: the features that pass the pre-skip, the block count of every ICP
    iteration, the pose."""
    import os
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Map, Point_cloud_registration
    here = os.path.dirname(__file__)
    g, s = np.load(os.path.join(here, "golden", "golden_r2.npz")), np.load(os.path.join(here, "golden", "golden_small.npz"))
    m = Map(ctx, s["map_corner"], s["map_surf"])
    for which, name in ((1, "surf"), (0, "corner")):
        ki, kd = m.nearestKSearch(which, s["knn_q"])
        assert np.array_equal(ki, g[f"flann_idx_{name}"]) and np.array_equal(kd, g[f"flann_d2_{name}"]), name
    m2 = Map(ctx, g["cap_map_corner"], g["cap_map_surf"])
    reg = Point_cloud_registration(ctx, maximum_allow_residual_block=int(g["cap"]), rng_seed=int(g["cap_seed"]))
    reg.set_pose(g["cap_guess_q"], g["cap_guess_t"])
    typ, a3, v3, ca, sa = reg.build_blocks(m2, g["cap_feat_corner"], g["cap_feat_surf"])
    assert np.array_equal(np.nonzero(typ)[0], g["cap_slots"]) and (ca, sa) == (int(g["cap_corner_avail"]), int(g["cap_surf_avail"]))
    st = reg.find_out_incremental_transfrom(m2, g["cap_feat_corner"], g["cap_feat_surf"])
    r = reg.result
    assert st == int(g["cap_status"]) and r.icp_iterations == int(g["cap_iters"]) and r.num_residual_blocks == int(g["cap_blocks"])
    assert np.linalg.norm(np.array(r.t_w_curr) - g["cap_t"]) < 1e-7 and S.quat_angle(np.array(r.q_w_curr), g["cap_q"]) < 1e-7
    L = capi.lib()
    k = 0
    for sd in (0, 3, -1):
        for it in (0, 5):
            for stream in (0, 1, 2):
                assert [L.ll_cap_uniform(sd, it, stream, i) for i in (0, 1, 7, 1000, 399999)] == list(g["cap_uniform"][k])
                k += 1


@pytest.mark.gpu
def test_ctx_warmup_leaves_results_untouched(oracle):
    """ll_ctx_warmup runs a toy registration (first-use costs paid up front; ll_mapper_create calls it): it must succeed on a fresh context, launch
    kernels, and a registration afterwards must return what it returns on a context that was never warmed."""
    from loam_livox_b200.registration import Context, Map, Point_cloud_registration
    mc, ms, fc, fs, pose = _mk(5000, 45000, 1000, 9000)
    guess = S.perturb_pose(pose, np.random.default_rng(3))
    out = []
    for warm in (True, False):
        c = Context(0, max_scan_points=100000, max_features=100000)
        if warm:
            l0 = c.launches(); c.warmup(); assert c.launches() > l0 + 5
        m = Map(c, mc, ms)
        reg = Point_cloud_registration(c); reg.set_pose(guess.q, guess.t)
        assert reg.find_out_incremental_transfrom(m, fc, fs) == 1
        r = reg.result
        out.append((r.icp_iterations, r.num_residual_blocks, tuple(r.q_w_curr), tuple(r.t_w_curr), r.final_cost))
        m.close() if hasattr(m, "close") else None
        c.close()
    assert out[0] == out[1]
    small = Context(0, max_scan_points=1000, max_features=100)   # smaller than the toy problem: a no-op, not an error
    small.warmup(); small.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode,window", [(0, 400), (0, 3), (1, 400)])
def test_streaming_mapper_reproduces_the_golden_track(ctx, mode, window):
    """The device mapper against the COMMITTED track of tests/golden/golden_stream.npz (oracle output, make_golden_stream.py; the oracle itself is pinned
    to it by tests/test_oracle.py): counts and ICP iterations exactly, pose < 1e-6 m / 1e-6 rad (bar 1e-4) after every one of the 14 scans."""
    import os
    import sys
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    import make_golden_stream as G
    want = np.load(os.path.join(os.path.dirname(__file__), "golden", "golden_stream.npz"))[f"track_m{mode}_w{window}"]
    gm = Laser_mapping(ctx, reg=capi.default_reg_state(mapping_init_accumulate_frames=G.INIT), matching_mode=mode, maximum_history_size=window)
    for k, raw in enumerate(G.scans()):
        res, st = gm.process_new_scan(raw, 100.0 + 0.1 * k)
        q, t, f = gm.pose()
        w = want[k]
        assert (res.status, f, st.n_corner, st.n_surf, st.map_corner, st.map_surf, st.appended_corner, st.appended_surf) == tuple(int(x) for x in w[:8]), k
        assert (res.icp_iterations if res.registered else 0) == int(w[8]), k
        dt, da = np.linalg.norm(t - w[13:16]), S.quat_angle(q, w[9:13])
        assert dt < 1e-4 and da < 1e-4, (k, dt, da)
        assert dt < 1e-6 and da < 1e-6, (k, dt, da)
