"""The spinning-lidar front end on the device (ll_spin_*, csrc/spin.cu) against the line-by-line oracle (oracle/orc_spin.hpp): all five
clouds and the per-point parity view bit for bit, on constructed edges and generated VLP-16 / HDL-64 scans."""
import ctypes as C

import numpy as np
import pytest

import spin_cases as SC
from loam_livox_b200 import capi, synthetic as S
from loam_livox_b200.registration import Context, Laser_feature, Map
from oracle.spin_oracle import CLOUDS, SpinExtractor

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sctx():
    c = Context(0, max_scan_points=20000, max_features=200000)
    yield c
    c.close()


@pytest.fixture(scope="module")
def fronts(sctx):
    f = {16: Laser_feature(sctx, 16), 64: Laser_feature(sctx, 64)}
    yield f
    for v in f.values():
        v.close()


def _check(front, scan_line, raw, device_input=None):
    o = SpinExtractor(scan_line)
    want = o.extract(raw)
    front.extract(raw if device_input is None else device_input)
    for k, name in enumerate(CLOUDS):
        got = front.cloud(k)
        assert got.shape == want[name].shape, (name, got.shape, want[name].shape)
        assert np.array_equal(got.view(np.uint32), want[name].view(np.uint32)), name
    for a, b, name in zip(front.point_info(), o.point_info(), ("ring", "curvature", "picked", "label")):
        assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32)), name
    return want


@pytest.mark.parametrize("name", sorted(SC.edge_cases()))
def test_edges_bit_exact(fronts, name):
    scan_line, raw = SC.edge_cases()[name]
    _check(fronts[scan_line], scan_line, raw)


@pytest.mark.parametrize("scan_line,n_az,scene,seed", [(16, 1800, "room", 1), (16, 1800, "open", 2), (64, 2080, "room", 3), (64, 2080, "open", 4)])
def test_generated_scans_bit_exact(fronts, scan_line, n_az, scene, seed):
    rng = np.random.default_rng(seed)
    raw = S.make_spinning_scan(scan_line, n_azimuth=n_az, scene=scene, seed=seed, start_azimuth_deg=rng.uniform(-180, 180), nan_frac=0.01, near_frac=0.005)
    want = _check(fronts[scan_line], scan_line, raw)
    assert len(want["sharp"]) > 0 and len(want["flat"]) > 0 and len(want["less_flat"]) > 0
    n_chains, longest = fronts[scan_line].chains()
    assert 1 <= n_chains <= 6 * scan_line and longest > 0


def test_input_formats(sctx, fronts):
    import torch
    raw = S.make_spinning_scan(16, n_azimuth=900, seed=5, nan_frac=0.01)
    want = _check(fronts[16], 16, raw)
    # pcl::PointXYZI records
    pcl = np.zeros((raw.shape[0], 8), np.float32); pcl[:, :3] = raw[:, :3]; pcl[:, 4] = raw[:, 3]
    _check(fronts[16], 16, raw, device_input=pcl)
    # a device cloud
    d = torch.from_numpy(raw).cuda()
    torch.cuda.synchronize()
    fronts[16].extract(d.data_ptr(), where=capi.LL_DEVICE, n=raw.shape[0], fmt=capi.LL_FMT_XYZI16)
    for k, name in enumerate(CLOUDS):
        assert np.array_equal(fronts[16].cloud(k).view(np.uint32), want[name].view(np.uint32)), name
    # a Velodyne PointCloud2 payload: x y z intensity(float32) ring(uint16) time(float32), 22-byte records
    rec = np.zeros(raw.shape[0], dtype=np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("intensity", "<f4"), ("ring", "<u2"), ("time", "<f4")]))
    for i, f in enumerate(("x", "y", "z", "intensity")):
        rec[f] = raw[:, i]
    rec["ring"] = 7
    sctx.set_point_layout(22, 0, 4, 8, 12, capi.LL_I_FLOAT32)
    try:
        fronts[16].extract_from_pointcloud2(rec.tobytes(), raw.shape[0])
    finally:
        sctx.set_point_layout(16)
    for k, name in enumerate(CLOUDS):
        assert np.array_equal(fronts[16].cloud(k).view(np.uint32), want[name].view(np.uint32)), name


def test_refusals(sctx):
    cfg = capi.default_spin_cfg(scan_line=32)
    h = C.c_void_p()
    assert sctx._lib.ll_spin_create(sctx.h, C.byref(cfg), C.byref(h)) == capi.LL_ERR_INVALID
    small = Laser_feature(sctx, 16, max_points=1000)
    raw = S.make_spinning_scan(16, n_azimuth=60, seed=9)
    small.extract(raw)
    before = [small.cloud(k) for k in range(5)]
    big = S.make_spinning_scan(16, n_azimuth=63, seed=10)   # 1008 points
    counts = (C.c_size_t * 5)()
    assert sctx._lib.ll_spin_extract(small.h, big.ctypes.data, big.shape[0], capi.LL_FMT_XYZI16, capi.LL_HOST, counts) == capi.LL_ERR_CAPACITY
    for k in range(5):
        assert np.array_equal(small.cloud(k).view(np.uint32), before[k].view(np.uint32))
    small.close()


def test_deterministic_across_runs_and_contexts(fronts):
    raw = S.make_spinning_scan(64, n_azimuth=2080, seed=21, nan_frac=0.01, start_azimuth_deg=123.0)
    fronts[64].extract(raw)
    first = [fronts[64].cloud(k) for k in range(5)]
    fronts[64].extract(raw)
    again = [fronts[64].cloud(k) for k in range(5)]
    ctx2 = Context(0, max_scan_points=1000, max_features=1000)
    other = Laser_feature(ctx2, 64, max_points=200000)
    other.extract(raw)
    third = [other.cloud(k) for k in range(5)]
    other.close(); ctx2.close()
    for a, b, c in zip(first, again, third):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)) and np.array_equal(a.view(np.uint32), c.view(np.uint32))


def test_register_device_features_against_room_map(sctx, fronts, oracle):
    """less sharp and less flat stay on the device and go straight into ll_register against the room map."""
    pose = S.Pose(S.quat_from_euler(0.0, 0.0, 0.05), np.array([0.3, 0.2, 0.1]))
    raw = S.make_spinning_scan(16, pose=pose, n_azimuth=1800, seed=31, nan_frac=0.01)
    mc, ms = S.make_map(5000, 45000)
    m = Map(sctx, mc, ms)
    guess = S.perturb_pose(pose, np.random.default_rng(0), dt=0.05, dang_deg=1.0)
    f = fronts[16]
    f.extract(raw)
    pc, nc = f.device_cloud(capi.LL_SPIN_LESS_SHARP)
    ps, ns = f.device_cloud(capi.LL_SPIN_LESS_FLAT)
    st = capi.default_reg_state(q_w_last=guess.q, t_w_last=guess.t, q_w_curr=guess.q, t_w_curr=guess.t)
    res = capi.RegResult()
    sctx.check(sctx._lib.ll_register(sctx.h, m.h, pc, nc, ps, ns, capi.LL_FMT_XYZI16, capi.LL_DEVICE, C.byref(st), C.byref(res)))
    o = SpinExtractor(16).extract(raw)
    p = oracle.default_params(q_w_last=guess.q, t_w_last=guess.t, q_w_curr=guess.q, t_w_curr=guess.t)
    ost, ores = oracle.register(mc, oracle.KdTree(mc), ms, oracle.KdTree(ms), o["less_sharp"], o["less_flat"], p)
    dt = float(np.linalg.norm(np.array(res.t_w_curr) - np.array(ores.t_w_curr)))
    da = S.quat_angle(np.array(res.q_w_curr), np.array(ores.q_w_curr))
    assert res.status == ost and dt < 1e-4 and da < 1e-4, (dt, da)
    assert np.linalg.norm(np.array(res.t_w_curr) - pose.t) < np.linalg.norm(guess.t - pose.t)
    assert S.quat_angle(np.array(res.q_w_curr), pose.q) < S.quat_angle(guess.q, pose.q)
    m.release()
