"""The piecewise frame on the device (ll_mapper_process_frame: every piece of a sensor frame registered as a scan of its own, odom_mode 1 of the
shipped configs) against the oracle's composition of the same steps (tests/piecewise_oracle.py), piece by piece; and the segmented VoxelGrid
(ll_voxel_downsample_segments) bit for bit against oracle.voxel_grid per segment."""
import ctypes as C
import os
import sys
import zlib

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from loam_livox_b200 import synthetic as S  # noqa: E402
import piecewise_oracle as PO  # noqa: E402

N = 24000


def pipeline(pieces=3):
    from loam_livox_b200 import capi
    return capi.PipelineCfg(pieces=pieces, use_piece=0, extractor_leaf_corner=0.1, extractor_leaf_surf=0.2, mapping_leaf_corner=0.1, mapping_leaf_surf=0.4, whole_frame=1)


def pair(ctx, oracle, pieces=3, mode=0, window=400, init=3, **reg):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping
    gm = Laser_mapping(ctx, reg=capi.default_reg_state(mapping_init_accumulate_frames=init, **reg), pipeline=pipeline(pieces), matching_mode=mode, maximum_history_size=window)
    om = oracle.Mapper(oracle.default_params(mapping_init_accumulate_frames=init, num_threads=4, **reg), threads=4, matching_mode=mode, maximum_history_size=window)
    return gm, om


def check_frame(gm, om, heads, stamps, pieces, odom_mode=1):
    """One frame on both sides: the same pieces published, and per piece status, registration, counts, ICP iterations and pose."""
    got = gm.process_new_frame(heads, stamps, odom_mode)
    want = PO.process_frame(om, heads, stamps, pieces, odom_mode)
    assert len(got) == len(want)
    for i, ((res, st), (ost, oq, ot, L)) in enumerate(zip(got, want)):
        assert res.status == ost, i
        assert (st.n_corner, st.n_surf) == (L["n_corner"], L["n_surf"]), i
        assert (st.map_corner, st.map_surf) == (L["map_corner"], L["map_surf"]), i
        if ost:
            assert (st.appended_corner, st.appended_surf) == (L["appended_corner"], L["appended_surf"]), i
        ores = L["res"]
        assert res.registered == (1 if ores is not None and ores.registered else 0), i
        if res.registered:
            assert res.icp_iterations == ores.icp_iterations, i
        assert np.linalg.norm(np.array(res.t_w_curr) - ot) < 1e-4 and S.quat_angle(np.array(res.q_w_curr), oq) < 1e-4, i
    assert gm.pose()[2] == om.frame_index
    return got, want


def raw_call(gm, heads, stamps, odom_mode=1, cap=16):
    """ll_mapper_process_frame directly: (status, *n_pieces, results)."""
    from loam_livox_b200 import capi
    k = len(heads)
    arrs = [np.ascontiguousarray(h, np.float32) for h in heads]
    ptrs = (C.c_void_p * k)(*[a.ctypes.data for a in arrs])
    sizes = (C.c_size_t * k)(*[a.shape[0] for a in arrs])
    st = (C.c_double * k)(*stamps)
    res, stats, n = (capi.RegResult * max(cap, 1))(), (capi.MapperStats * max(cap, 1))(), C.c_int(-1)
    status = gm.ctx._lib.ll_mapper_process_frame(gm.h, k, ptrs, sizes, capi.LL_FMT_XYZI16, capi.LL_HOST, st, odom_mode, res, stats, cap, C.byref(n))
    return status, n.value, [res[i] for i in range(max(n.value, 0))]


def few_petals(raw, oracle, petals):
    ex = oracle.Extractor()
    n = raw.shape[0]
    for m in range(n // 40, n, n // 200):
        if ex.extract(raw[:m], 100.0) == petals:
            return raw[:m].copy()
    raise AssertionError(petals)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,window", [(0, 400), (0, 3), (1, 400)])
def test_piecewise_stream_matches_the_oracle(ctx, oracle, mode, window):
    """8 frames x 3 pieces, every piece a scan of its own (window 3 pops): per piece exactly the oracle's counts, status and ICP iterations,
    pose within 1e-4 m / 1e-4 rad; the frame index counts pieces."""
    gm, om = pair(ctx, oracle, mode=mode, window=window)
    for k, pose in enumerate(S.trajectory(n_scans=8, n_static=2, speed=1.0)):
        check_frame(gm, om, [S.make_scan(N, pose, seed=S.SEED + 700 + k)], [100.0 + 0.1 * k], 3)
    assert gm.pose()[2] == 24


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["track_m0_w400", "track_m0_w3", "track_m1_w400", "track_heads3_p2"])
def test_piecewise_stream_reproduces_the_golden_track(ctx, name):
    """The device mapper against the committed oracle track of tests/golden/golden_pieces.npz: counts and ICP iterations exactly, pose 1e-6."""
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    import make_golden_pieces as G
    want = np.load(os.path.join(os.path.dirname(__file__), "golden", "golden_pieces.npz"))[name]
    heads3 = name == "track_heads3_p2"
    mode, window = (0, 400) if heads3 else (int(name[7]), int(name.split("_w")[1]))
    pieces = G.HEADS_PIECES if heads3 else G.PIECES
    gm = Laser_mapping(ctx, reg=capi.default_reg_state(mapping_init_accumulate_frames=G.INIT), pipeline=pipeline(pieces), matching_mode=mode, maximum_history_size=window)
    rows = []
    for k, heads in enumerate(G.head_frames() if heads3 else G.frames()):
        for res, st in gm.process_new_frame(heads, G.stamps(k, len(heads))):
            icp = res.icp_iterations if res.registered else 0
            rows.append([res.status, 0, st.n_corner, st.n_surf, st.map_corner, st.map_surf, st.appended_corner, st.appended_surf, icp] + list(res.q_w_curr) + list(res.t_w_curr))
    got = np.array(rows)
    assert got.shape == want.shape
    assert np.array_equal(got[:, [0, 2, 3, 4, 5, 6, 7, 8]], want[:, [0, 2, 3, 4, 5, 6, 7, 8]])
    assert np.abs(got[:, 9:] - want[:, 9:]).max() < 1e-6
    assert gm.pose()[2] == int(want[-1, 1])


@pytest.mark.gpu
def test_shipped_init_gate_counts_pieces(ctx, oracle):
    """mapping/init_accumulate_frames = 50 counts pieces: with 3 pieces per frame the first ICP is piece 0 of frame 17 (frame index 51)."""
    gm, om = pair(ctx, oracle, init=50)
    first = None
    for k, pose in enumerate(S.trajectory(n_scans=18, n_static=18, speed=1.0)):
        got, _ = check_frame(gm, om, [S.make_scan(N, pose, seed=S.SEED + 800 + k)], [100.0 + 0.1 * k], 3)
        for i, (res, _) in enumerate(got):
            if res.registered and first is None:
                first = (k, i)
    assert first == (17, 0)


@pytest.mark.gpu
def test_odom_mode_0_registers_what_frame_to_pose_registers(ctx, oracle):
    """odom_mode 0: one registration per frame, on exactly the features ll_frame_to_pose registers with use_piece 0 (bit for bit)."""
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping, Map, features_to_pointcloud2, frame_to_pose
    poses = S.trajectory(n_scans=3, n_static=1, speed=1.0)
    frames = [[S.make_scan(N, p, seed=S.SEED + 900 + k)] for k, p in enumerate(poses)]
    stamps = [[100.0 + 0.1 * k] for k in range(3)]
    gm = Laser_mapping(ctx, reg=capi.default_reg_state(mapping_init_accumulate_frames=-1), pipeline=pipeline(3))
    for k in range(2):
        out = gm.process_new_frame(frames[k], stamps[k], odom_mode=0)
        assert len(out) == 1 and gm.pose()[2] == k + 1
    assert out[0][0].registered == 1
    mine = (features_to_pointcloud2(ctx, 0), features_to_pointcloud2(ctx, 1))
    gm.close()
    ctx._lib.ll_extract_reset(ctx.h)
    mc, ms = S.make_map(5000, 45000)
    m = Map(ctx, mc, ms)
    pc = capi.PipelineCfg(pieces=3, use_piece=0, extractor_leaf_corner=0.1, extractor_leaf_surf=0.2, mapping_leaf_corner=0.1, mapping_leaf_surf=0.4, whole_frame=0)
    for k in range(2):
        st = capi.default_reg_state(q_w_last=poses[k].q, t_w_last=poses[k].t, q_w_curr=poses[k].q, t_w_curr=poses[k].t)
        res, nc, nsf = frame_to_pose(ctx, m, frames[k], stamps[k], pc, st)
    assert (nc, nsf) == (out[0][1].n_corner, out[0][1].n_surf)
    assert (features_to_pointcloud2(ctx, 0), features_to_pointcloud2(ctx, 1)) == mine
    m.release()


@pytest.mark.gpu
def test_motion_deblur_registers_one_piece_with_petal_bounds(ctx, oracle):
    """if_motion_deblur = 1: one piece per frame, cut at the petal bounds of piece_bounds(1) (not 0 ... 1), registered with the deblur
    functors; per frame against the oracle."""
    gm, om = pair(ctx, oracle, init=2, if_motion_deblur=1)
    for k, pose in enumerate(S.trajectory(n_scans=6, n_static=2, speed=1.0)):
        raw = S.make_scan(N, pose, seed=S.SEED + 1000 + k)
        got, want = check_frame(gm, om, [raw], [100.0 + 0.1 * k], 1)
        assert len(got) == 1
    ex = oracle.Extractor()
    ex.extract(raw, 100.0)
    start, end = ex.piece_bounds(1)
    assert (start[0], end[0]) != (0.0, 1.0)
    assert got[0][0].registered == 1


@pytest.mark.gpu
def test_mid100_frames_with_dropped_heads(ctx, oracle):
    """3 heads x 2 pieces over several frames; one frame with a head of <= 5 petals (it contributes nothing) and one where every head has
    <= 5 petals (*n_pieces == 0, frame index unchanged)."""
    gm, om = pair(ctx, oracle, pieces=2)
    poses = S.trajectory(n_scans=6, n_static=2, speed=1.0)
    for k, pose in enumerate(poses):
        heads = S.make_triple_scan(3 * 16000, pose, seed=S.SEED + 1100 + 3 * k)
        if k == 3:
            heads[1] = heads[1][: heads[1].shape[0] // 8]
        if k == 4:
            heads = [h[:200] for h in heads]
            before = gm.pose()
            status, n, _ = raw_call(gm, heads, [100.0 + 0.1 * k] * 3)
            assert status == 0 and n == 0
            after = gm.pose()
            assert after[2] == before[2] and np.array_equal(after[0], before[0]) and np.array_equal(after[1], before[1])
            assert PO.process_frame(om, heads, [100.0 + 0.1 * k] * 3, 2) == []
            continue
        got, _ = check_frame(gm, om, heads, [100.0 + 0.1 * k] * 3, 2)
        assert len(got) == 2


@pytest.mark.gpu
def test_overlapping_pieces(ctx, oracle):
    """16 pieces of a frame with 6 ... 8 petals: the bounds clamp, pieces overlap and the same points go to several pieces (others are empty);
    per piece feature, map and append counts against the oracle.  Below the init gate: a piece without features cannot be registered."""
    gm, om = pair(ctx, oracle, pieces=16, init=100)
    for k, pose in enumerate(S.trajectory(n_scans=3, n_static=2, speed=1.0)):
        raw = few_petals(S.make_scan(N, pose, seed=S.SEED + 1200 + k), oracle, 6 + k)
        got, _ = check_frame(gm, om, [raw], [100.0 + 0.1 * k], 16)
        counts = [(st.n_corner, st.n_surf) for _, st in got]
        assert len(set(counts)) < len(counts)   # repeated pieces
    assert gm.pose()[2] == 48


@pytest.mark.gpu
def test_rejected_piece_mid_frame(ctx, oracle):
    """A tight max_final_cost rejects registered pieces: the status sequence equals the oracle's, the pose is unchanged after a rejection and
    the next pieces of the frame continue from it."""
    gm, om = pair(ctx, oracle, init=3, max_final_cost=1e-7)
    statuses = []
    for k, pose in enumerate(S.trajectory(n_scans=4, n_static=1, speed=1.0)):
        before = gm.pose()
        got, _ = check_frame(gm, om, [S.make_scan(N, pose, seed=S.SEED + 1300 + k)], [100.0 + 0.1 * k], 3)
        for res, _ in got:
            statuses.append(res.status)
            if res.status == 0:
                assert np.array_equal(np.array(res.q_w_curr), before[0]) and np.array_equal(np.array(res.t_w_curr), before[1])
    assert 0 in statuses and gm.pose()[2] == 12


@pytest.mark.gpu
def test_errors(oracle):
    """LL_ERR_CAPACITY at piece 1 leaves the oracle's state after piece 0 (*n_pieces == 1); cap too small, a bad odom_mode and bad pieces are
    LL_ERR_INVALID with nothing changed."""
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Context, Laser_mapping
    # a frame whose piece 1 has more features than piece 0
    for seed in range(S.SEED + 1400, S.SEED + 1440):
        raw = S.make_scan(N, seed=seed)
        parts, _ = PO.frame_pieces(oracle.Extractor(), [raw], [100.0], 3)
        f = [oracle.voxel_grid(oracle.voxel_grid(c, 0.1), 0.1).shape[0] + oracle.voxel_grid(oracle.voxel_grid(s, 0.2), 0.4).shape[0] for c, s, _ in parts]
        if f[1] > f[0]:
            break
    assert f[1] > f[0]
    small = Context(0, max_scan_points=N, max_features=f[0])
    try:
        gm = Laser_mapping(small, reg=capi.default_reg_state(mapping_init_accumulate_frames=3), pipeline=pipeline(3))
        om = oracle.Mapper(oracle.default_params(mapping_init_accumulate_frames=3, num_threads=4), threads=4)
        status, n, res = raw_call(gm, [raw], [100.0])
        assert status == capi.LL_ERR_CAPACITY and n == 1
        PO.process_frame(om, [raw], [100.0], 3, odom_mode=0)
        q, t, fi = gm.pose()
        assert fi == om.frame_index == 1 and np.abs(t - om.t).max() < 1e-9 and np.abs(q - om.q).max() < 1e-9
        for args in (dict(cap=2), dict(odom_mode=2), dict(odom_mode=-1)):
            status, n, _ = raw_call(gm, [raw], [100.1], **args)
            assert status == capi.LL_ERR_INVALID and n == 0 and gm.pose()[2] == 1, args
        gm.close()
        for p in (0, 17):
            gm = Laser_mapping(small, pipeline=pipeline(p))
            status, n, _ = raw_call(gm, [raw], [100.2])
            assert status == capi.LL_ERR_INVALID and n == 0 and gm.pose()[2] == 0
            gm.close()
    finally:
        small.close()


# ---------------------------------------------------------------------------------------------- segmented VoxelGrid
def _segments_case(name, rng):
    """(cloud, seg_end, leaf) for one edge case."""
    def blob(n, scale=5.0, off=0.0):
        p = rng.uniform(-scale, scale, (n, 4)).astype(np.float32)
        p[:, :3] += off
        p[:, 3] = rng.uniform(0, 100, n)
        return p
    if name.startswith("uniform"):
        k = int(name[7:])
        sizes = rng.integers(200, 3000, k)
        segs = [blob(int(s), off=float(j)) for j, s in enumerate(sizes)]
        leaf = 0.4
    elif name == "empty_and_nan":
        nan = blob(300); nan[:, :3] = np.nan
        segs = [blob(1000), np.zeros((0, 4), np.float32), nan, blob(700), np.zeros((0, 4), np.float32)]
        leaf = 0.2
    elif name == "overflow_between":
        far = blob(500, scale=1.0); far[0, :3] = -1.0e6; far[1, :3] = 1.0e6
        segs = [blob(800), far, blob(900)]
        leaf = 0.01
    elif name == "same_coordinates":
        a = blob(1500)
        segs = [a, a.copy(), a[::-1].copy()]
        leaf = 0.5
    elif name == "faces":
        g = rng.integers(-20, 20, (3000, 3)).astype(np.float32) * np.float32(0.25)
        p = np.concatenate([g, rng.uniform(0, 1, (3000, 1)).astype(np.float32)], axis=1)
        segs = [p[:1000], p[1000:2100], p[2100:]]
        leaf = 0.25
    elif name == "block_edges":
        segs = [blob(n) for n in (255, 256, 257, 1, 511, 512, 513, 33 * 1024 + 7, 70000)]
        leaf = 0.3
    elif name == "one_large":
        segs = [blob(300000, scale=30.0)]
        leaf = 0.2
    cloud = np.concatenate(segs).astype(np.float32)
    ends = np.cumsum([s.shape[0] for s in segs]).astype(np.uint64)
    return cloud, ends, np.float32(leaf), segs


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["uniform1", "uniform2", "uniform3", "uniform16", "empty_and_nan", "overflow_between", "same_coordinates", "faces",
                                  "block_edges", "one_large"])
def test_segmented_voxel_grid_matches_per_segment_voxel_grid(ctx, oracle, name):
    """ll_voxel_downsample_segments: each segment's output is bit for bit oracle.voxel_grid of that segment alone -- empty and all-NaN segments,
    an int32-overflow pass-through segment between normal ones, the same coordinates in adjacent segments (never merged), points on voxel faces,
    sizes around the 256-thread blocks and past the min/max kernel's capped grid."""
    from loam_livox_b200.registration import voxel_grid_segments
    cloud, ends, leaf, segs = _segments_case(name, np.random.default_rng(zlib.crc32(name.encode())))
    got = voxel_grid_segments(ctx, cloud, ends, leaf)
    assert len(got) == len(segs)
    for k, (g, s) in enumerate(zip(got, segs)):
        want = oracle.voxel_grid(s, leaf) if s.shape[0] else np.zeros((0, 4), np.float32)
        assert g.shape == want.shape and g.tobytes() == want.tobytes(), (name, k)
