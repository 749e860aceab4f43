"""The streaming mapper on spinning-lidar sweeps (ll_mapper_process_sweep / _sweeps, DESIGN.md §4.7.1) against the oracle composition of the
reference's remapped Velodyne pipeline (tests/spin_mapper_oracle.py): per-sweep parity in both matching modes, HDL-64 and motion deblur, the
golden track, sequences against single calls, edges inside a stream, refusals that change nothing, input formats, the checkpoint, loop closure
and recovery."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from loam_livox_b200 import synthetic as S  # noqa: E402
import make_golden_spin as G  # noqa: E402
import spin_mapper_oracle as SMO  # noqa: E402

pytestmark = pytest.mark.gpu

STAT_INTS = ("n_corner", "n_surf", "map_corner", "map_surf", "cells_in_fov_corner", "cells_in_fov_surf", "appended_corner", "appended_surf")


@pytest.fixture(scope="module")
def ctxs():
    from loam_livox_b200.registration import Context
    cs = [Context(0, max_scan_points=60000, max_features=400000) for _ in range(2)]
    yield cs
    for c in cs:
        c.close()


@pytest.fixture(scope="module")
def fronts(ctxs):
    from loam_livox_b200.registration import Laser_feature
    f = [{16: Laser_feature(c, 16), 64: Laser_feature(c, 64)} for c in ctxs]
    yield f
    for d in f:
        for v in d.values():
            v.close()


def _mapper(ctx, mode=0, window=400, init=G.INIT, p0=None, **reg):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping
    if p0 is not None:
        reg = dict(reg, q_w_last=p0.q, t_w_last=p0.t, q_w_curr=p0.q, t_w_curr=p0.t)
    return Laser_mapping(ctx, reg=capi.default_reg_state(mapping_init_accumulate_frames=init, **reg), matching_mode=mode, maximum_history_size=window)


def _b(x):
    return np.array(list(x) if isinstance(x, C.Array) else [x]).tobytes()


def entry(res, st):
    """every non-timing field of the result, every integer field of the stats"""
    from loam_livox_b200 import capi
    return tuple(_b(getattr(res, f)) for f, _ in capi.RegResult._fields_ if not f.startswith("gpu_ms")) + tuple(getattr(st, f) for f in STAT_INTS)


def state(gm):
    q, t, f = gm.pose()
    return q.tobytes(), t.tobytes(), f


def singles(gm, front, raws, **kw):
    return [entry(*gm.process_new_sweep(front, r, **kw)) for r in raws]


def seq(gm, front, raws, split=None, **kw):
    out, i = [], 0
    for n in split or [len(raws)]:
        sub = {k: (v[i:i + n] if k == "ns" else v) for k, v in kw.items()}
        out += [entry(r, s) for r, s in gm.process_new_sweeps(front, raws[i:i + n], **sub)]
        i += n
    return out


def check_sweep(res, st, gm, want, frame_index):
    ost, oq, ot, L = want
    assert res.status == ost
    assert (st.n_corner, st.n_surf) == (L["n_corner"], L["n_surf"])
    assert (st.map_corner, st.map_surf) == (L["map_corner"], L["map_surf"])
    if ost:
        assert (st.appended_corner, st.appended_surf) == (L["appended_corner"], L["appended_surf"])
    ores = L["res"]
    assert res.registered == (1 if ores is not None and ores.registered else 0)
    if res.registered:
        assert res.icp_iterations == ores.icp_iterations
    assert np.linalg.norm(np.array(res.t_w_curr) - ot) < 1e-4 and S.quat_angle(np.array(res.q_w_curr), oq) < 1e-4
    assert gm.pose()[2] == frame_index


def vlp(n, seed, **kw):
    poses = S.trajectory(n_scans=n, n_static=2, speed=1.0)
    return [S.make_spinning_scan(16, p, seed=seed + k, **kw) for k, p in enumerate(poses)]


# ---------------------------------------------------------------------------------------------- 1. parity with the composition
CASES = {"vlp16_m0_w400": (16, 0, 400, {}), "vlp16_m0_w3": (16, 0, 3, {}), "vlp16_m1_w400": (16, 1, 400, {}), "hdl64_open": (64, 0, 400, {}),
         "vlp16_deblur": (16, 0, 400, dict(if_motion_deblur=1))}


@pytest.mark.parametrize("name", list(CASES))
def test_parity_with_the_composition(ctxs, fronts, oracle, name):
    """Per sweep: status, feature, map and appended counts and ICP iterations equal the composition's, the pose within 1e-4 m / 1e-4 rad, and
    the frame index counts sweeps."""
    scan_line, mode, window, reg = CASES[name]
    raws = G.hdl_sweeps()[0] if scan_line == 64 else vlp(10, S.SEED + 900)
    gm = _mapper(ctxs[0], mode, window, **reg)
    om = G.oracle_mapper(scan_line, mode, window, **reg)
    try:
        registered = []
        for k, raw in enumerate(raws):
            res, st = gm.process_new_sweep(fronts[0][scan_line], raw)
            check_sweep(res, st, gm, om.process_sweep(raw), k + 1)
            registered.append(res.registered)
        assert any(registered)
    finally:
        gm.close()


# ---------------------------------------------------------------------------------------------- 2. the golden track
@pytest.mark.parametrize("name", [f"track_vlp16_m{m}_w{w}" for m, w in G.CASES] + ["track_hdl64_open"])
def test_golden_track(ctxs, fronts, name):
    """tests/golden/golden_spin.npz through one process_new_sweeps call: counts and ICP iterations exactly, pose within 1e-6."""
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "golden_spin.npz"))[name]
    if name == "track_hdl64_open":
        scan_line, mode, window, raws = 64, 0, 400, G.hdl_sweeps()[0]
    else:
        scan_line, raws = 16, G.vlp_sweeps()[0]
        mode, window = (int(x[1:]) for x in name.split("_")[2:])
    gm = _mapper(ctxs[1], mode, window)
    try:
        out = gm.process_new_sweeps(fronts[1][scan_line], raws)
        rows = [[r.status, 0, s.n_corner, s.n_surf, s.map_corner, s.map_surf, s.appended_corner if r.status else 0, s.appended_surf if r.status else 0,
                 r.icp_iterations if r.registered else 0] + list(r.q_w_curr) + list(r.t_w_curr) for r, s in out]
        got = np.array(rows)
        cols = [0, 2, 3, 4, 5, 6, 7, 8]
        assert np.array_equal(got[:, cols], gold[:, cols])
        assert np.abs(got[:, 9:] - gold[:, 9:]).max() < 1e-6
        assert gm.pose()[2] == int(gold[-1, 1])
    finally:
        gm.close()


# ---------------------------------------------------------------------------------------------- 3. sequences
@pytest.mark.parametrize("mode,window", [(0, 3), (1, 400)])
def test_sequences_equal_single_calls(ctxs, fronts, mode, window):
    """process_new_sweeps in every split equals the single calls: entries, integer stats, pose and save() bytes; afterwards the spin handle's
    clouds are the last sweep's, bit for bit those of ll_spin_extract."""
    from loam_livox_b200.registration import Laser_feature
    raws = vlp(9, S.SEED + 950)
    ga, gb = _mapper(ctxs[0], mode, window), _mapper(ctxs[1], mode, window)
    try:
        la, lb = ctxs[0].launches(), ctxs[1].launches()
        want = singles(ga, fronts[0][16], raws)
        got = seq(gb, fronts[1][16], raws, split=[4, 1, 4])
        assert got == want
        assert ctxs[0].launches() - la == ctxs[1].launches() - lb
        assert state(ga) == state(gb) and ga.save() == gb.save()
        ref = Laser_feature(ctxs[0], 16)
        ref.extract(raws[-1])
        for k in range(5):
            a, b = fronts[1][16].cloud(k), ref.cloud(k)
            assert a.shape == b.shape and a.tobytes() == b.tobytes(), k
        ref.close()
    finally:
        ga.close(); gb.close()


# ---------------------------------------------------------------------------------------------- 4. edges inside a stream
def _edge_stream(seed):
    raws = vlp(10, seed)
    few = np.full((40, 4), np.nan, np.float32)
    few[:4] = raws[0][:4]
    edges = [np.zeros((0, 4), np.float32), np.zeros((0, 4), np.float32), np.full((100, 4), np.nan, np.float32), few]
    return raws[:1] + edges[:1] + raws[1:3] + edges[1:2] + raws[3:4] + edges[2:3] + raws[4:5] + edges[3:] + raws[5:], edges


def test_edges_inside_a_stream(ctxs, fronts, oracle):
    """An empty sweep, an all-NaN sweep and a sweep with fewer than 5 kept points, each followed by normal sweeps, against the composition
    sweep by sweep: before the registration gate (mapping_init_accumulate_frames 10) they go through the step with 0 features and append
    nothing; the sweeps after them register as the composition's do.  The sequence call equals the single calls."""
    from oracle import oracle as O
    init = 10
    stream, edges = _edge_stream(S.SEED + 1000)
    gm, gb = _mapper(ctxs[0], init=init), _mapper(ctxs[1], init=init)
    om = SMO.SpinMapper(16, params=O.default_params(mapping_init_accumulate_frames=init, num_threads=G.THREADS), threads=G.THREADS)
    try:
        want, registered = [], []
        for k, raw in enumerate(stream):
            res, st = gm.process_new_sweep(fronts[0][16], raw)
            check_sweep(res, st, gm, om.process_sweep(raw), k + 1)
            if any(raw is e for e in edges):
                assert k < init and (st.n_corner, st.n_surf, st.appended_corner, st.appended_surf) == (0, 0, 0, 0)
            registered.append(res.registered)
            want.append(entry(res, st))
        assert sum(registered) >= 3
        assert seq(gb, fronts[1][16], stream) == want and gm.save() == gb.save()
    finally:
        gm.close(); gb.close()


def test_empty_sweeps_past_the_gate(ctxs, fronts):
    """Past the registration gate an empty sweep is the empty registration of any scan: LL_ERR_NO_BLOCKS, the frame index counted, the pose
    kept, nothing appended.  The sequence call stops at it (done = f) and, resumed after it, gives the single calls' results and image."""
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import LoamLivoxError, SequenceError
    stream, edges = _edge_stream(S.SEED + 1050)
    gm, gb = _mapper(ctxs[0]), _mapper(ctxs[1])
    try:
        want, stops = [], []
        for k, raw in enumerate(stream):
            if any(raw is e for e in edges) and k + 1 > G.INIT:
                before = gm.pose()
                with pytest.raises(LoamLivoxError) as e:
                    gm.process_new_sweep(fronts[0][16], raw)
                assert f"status {capi.LL_ERR_NO_BLOCKS}" in str(e.value)
                q, t, f = gm.pose()
                assert f == k + 1 and q.tobytes() == before[0].tobytes() and t.tobytes() == before[1].tobytes()
                want.append(None)
                stops.append(k)
                continue
            want.append(entry(*gm.process_new_sweep(fronts[0][16], raw)))
        assert stops == [4, 6, 8]
        i = 0
        for f in stops:
            with pytest.raises(SequenceError) as e:
                gb.process_new_sweeps(fronts[1][16], stream[i:])
            assert e.value.status == capi.LL_ERR_NO_BLOCKS and e.value.done == f - i
            assert [entry(r, s) for r, s in e.value.results] == want[i:f]
            i = f + 1
        assert seq(gb, fronts[1][16], stream[i:]) == want[i:]
        assert state(gm) == state(gb) and gm.save() == gb.save()
    finally:
        gm.close(); gb.close()


def test_rejected_sweeps_against_the_composition(ctxs, fronts, oracle):
    """A tight max_final_cost rejects registered sweeps: the statuses equal the composition's, a rejected sweep leaves the pose as it was and
    the next sweeps continue from it."""
    raws = vlp(7, S.SEED + 1100)
    gm = _mapper(ctxs[0], max_final_cost=1e-7)
    om = G.oracle_mapper(16, 0, 400, max_final_cost=1e-7)
    try:
        statuses = []
        for k, raw in enumerate(raws):
            before = gm.pose()
            res, st = gm.process_new_sweep(fronts[0][16], raw)
            check_sweep(res, st, gm, om.process_sweep(raw), k + 1)
            statuses.append(res.status)
            if res.status == 0:
                assert np.array_equal(np.array(res.q_w_curr), before[0]) and np.array_equal(np.array(res.t_w_curr), before[1])
        assert 0 in statuses
    finally:
        gm.close()


# ---------------------------------------------------------------------------------------------- 5. refusals
def _sweeps_call(gm, front, raws, n=None):
    from loam_livox_b200 import capi
    arrs = [np.ascontiguousarray(r, np.float32) for r in raws]
    k = len(arrs)
    ptrs = (C.c_void_p * k)(*[a.ctypes.data for a in arrs])
    sizes = (C.c_size_t * k)(*[a.shape[0] for a in arrs])
    res, stats, done = (capi.RegResult * k)(), (capi.MapperStats * k)(), C.c_int(-1)
    st = gm.ctx._lib.ll_mapper_process_sweeps(gm.h, front.h, k if n is None else n, ptrs, sizes, capi.LL_FMT_XYZI16, capi.LL_HOST, res, stats, C.byref(done))
    return st, done.value


def test_refusals_change_nothing(ctxs, fronts):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Context, Laser_feature
    raws = vlp(6, S.SEED + 1200)
    gm = _mapper(ctxs[0])
    try:
        gm.process_new_sweeps(fronts[0][16], raws[:4])
        img, pose = gm.save(), state(gm)
        # a spin handle of another context
        assert _sweeps_call(gm, fronts[1][16], raws[4:]) == (capi.LL_ERR_INVALID, 0)
        res, st = capi.RegResult(), capi.MapperStats()
        a = np.ascontiguousarray(raws[4])
        assert gm.ctx._lib.ll_mapper_process_sweep(gm.h, fronts[1][16].h, a.ctypes.data, a.shape[0], capi.LL_FMT_XYZI16, capi.LL_HOST, C.byref(res),
                                                   C.byref(st)) == capi.LL_ERR_INVALID
        assert _sweeps_call(gm, fronts[0][16], raws[4:], n=0) == (capi.LL_ERR_INVALID, 0)
        assert gm.ctx._lib.ll_mapper_process_sweep(gm.h, fronts[0][16].h, a.ctypes.data, a.shape[0], 7, capi.LL_HOST, C.byref(res), C.byref(st)) == capi.LL_ERR_INVALID
        # a sweep over max_points anywhere in the sequence
        small = Laser_feature(ctxs[0], 16, max_points=20000)
        assert _sweeps_call(gm, small, [raws[4][:10000], raws[5]]) == (capi.LL_ERR_CAPACITY, 0)
        small.close()
        assert gm.save() == img and state(gm) == pose
    finally:
        gm.close()
    # loop closure on: sweeps of exactly max_scan_points run through loop closure (every point kept: the world-frame buffer and one append of
    # the full map are filled to the last point); one point more is refused up front
    S_ = 12000
    c = Context(0, max_scan_points=S_, max_features=60000)
    try:
        f = Laser_feature(c, 16)
        m = _mapper(c)
        m.set_loop_closure(**dict(SMALL, loop=dict(SMALL["loop"], minimum_keyframe_differen=100000)))
        many = vlp(8, S.SEED + 1250)
        m.process_new_sweeps(f, [r[:S_] for r in many])
        assert f.cloud(capi.LL_SPIN_FULL).shape[0] > S_ - 200
        log, _ = m.loop_log()
        assert [e for e in log if e.kind == capi.LL_LOOP_KEYFRAME]
        assert not [e for e in log if e.kind == capi.LL_LOOP_ERROR]
        img, lr = m.save(), m.loop_result()
        assert _sweeps_call(m, f, [raws[3][:S_], raws[4][:S_ + 1]]) == (capi.LL_ERR_CAPACITY, 0)
        assert m.save() == img and m.loop_result()["poses_ori"].tobytes() == lr["poses_ori"].tobytes()
        m.close(); f.close()
    finally:
        c.close()


def test_features_over_max_features_stop_the_sequence(ctxs):
    """Half sweeps fit max_features, a whole one does not: the sequence stops at it with done = f, the mapper as after the single calls up to
    f, and the run continues by either API to the same end."""
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Context, Laser_feature, LoamLivoxError, SequenceError
    poses = S.trajectory(n_scans=7, n_static=2, speed=1.0)
    raws = [S.make_spinning_scan(16, p, seed=S.SEED + 1300 + k, n_azimuth=900 if k != 3 else 1800, sweep_deg=180.0 if k != 3 else 360.0)
            for k, p in enumerate(poses)]
    cs = [Context(0, max_scan_points=60000, max_features=1600) for _ in range(2)]
    try:
        fs = [Laser_feature(c, 16) for c in cs]
        ga, gb = _mapper(cs[0]), _mapper(cs[1])
        want = singles(ga, fs[0], raws[:3])
        with pytest.raises(LoamLivoxError) as e:
            ga.process_new_sweep(fs[0], raws[3])
        assert f"status {capi.LL_ERR_CAPACITY}" in str(e.value)
        with pytest.raises(SequenceError) as e:
            gb.process_new_sweeps(fs[1], raws)
        assert e.value.status == capi.LL_ERR_CAPACITY and e.value.done == 3
        assert [entry(r, s) for r, s in e.value.results] == want
        assert state(ga) == state(gb) and ga.save() == gb.save()
        a = singles(ga, fs[0], raws[4:])
        b = seq(gb, fs[1], raws[4:])
        assert a == b and state(ga) == state(gb) and ga.save() == gb.save()
        ga.close(); gb.close()
        for f in fs:
            f.close()
    finally:
        for c in cs:
            c.close()


# ---------------------------------------------------------------------------------------------- 6. input formats
def _strided(raw, step=20):
    rec = np.zeros((raw.shape[0], step), np.uint8)
    rec[:, 0:12] = raw[:, :3].astype(np.float32).view(np.uint8).reshape(-1, 12)
    rec[:, 16:20] = raw[:, 3:4].astype(np.float32).view(np.uint8).reshape(-1, 4)
    return rec


def test_input_formats(ctxs, fronts):
    """PCL32 records, strided PointCloud2 records and device inputs give the XYZI16 host results, in single and sequence calls."""
    import torch
    from loam_livox_b200 import capi
    raws = vlp(6, S.SEED + 1400)

    def run(fn, arm=1):
        gm = _mapper(ctxs[arm])
        try:
            return fn(gm, fronts[arm][16]), gm.save()
        finally:
            gm.close()

    want = run(lambda g, f: singles(g, f, raws), 0)
    pcl = [np.concatenate([r[:, :3], np.zeros((r.shape[0], 1), np.float32), r[:, 3:4], np.zeros((r.shape[0], 3), np.float32)], axis=1) for r in raws]
    assert run(lambda g, f: seq(g, f, pcl, split=[2, 4])) == want
    assert run(lambda g, f: singles(g, f, pcl)) == want
    recs = [_strided(r) for r in raws]
    ctxs[1].set_point_layout(20, 0, 4, 8, 16, capi.LL_I_FLOAT32)
    try:
        assert run(lambda g, f: seq(g, f, recs, fmt=capi.LL_FMT_STRIDED, ns=[r.shape[0] for r in recs])) == want
    finally:
        ctxs[1].set_point_layout(16)
    dev = [torch.from_numpy(r).cuda() for r in raws]
    torch.cuda.synchronize()
    ptrs, ns = [d.data_ptr() for d in dev], [d.shape[0] for d in dev]
    assert run(lambda g, f: seq(g, f, ptrs, where=capi.LL_DEVICE, ns=ns, fmt=capi.LL_FMT_XYZI16)) == want
    assert run(lambda g, f: [entry(*g.process_new_sweep(f, p, where=capi.LL_DEVICE, n=n, fmt=capi.LL_FMT_XYZI16)) for p, n in zip(ptrs, ns)]) == want


# ---------------------------------------------------------------------------------------------- 7. checkpoint
def test_checkpoint_continues_bit_for_bit(ctxs, fronts):
    """Save mid-stream, load on the second context, continue both: equal entries and equal images."""
    from loam_livox_b200.registration import Laser_mapping
    raws = vlp(10, S.SEED + 1500)
    ga = _mapper(ctxs[0], 1, 400)
    try:
        ga.process_new_sweeps(fronts[0][16], raws[:5])
        gb = Laser_mapping.load(ctxs[1], ga.save())
        assert state(gb) == state(ga)
        a = seq(ga, fronts[0][16], raws[5:])
        b = singles(gb, fronts[1][16], raws[5:])
        assert a == b and state(ga) == state(gb) and ga.save() == gb.save()
        gb.close()
    finally:
        ga.close()


# ---------------------------------------------------------------------------------------------- 8. loop closure
SMALL = dict(scans_of_each_keyframe=6, scans_between_two_keyframe=2, reserve_map_points=1 << 21, reserve_history_points=1 << 21, reserve_keyframes=64,
             loop=dict(minimum_keyframe_differen=36, avail_ratio_plane=0.02, avail_ratio_line=0.005), map_alignment_inlier_threshold=0.35)


def _returning(n_out=40, step=0.15):
    xs = [0.3 + step * k for k in range(n_out)] + [0.3 + step * (n_out - 1 - k) for k in range(n_out)]
    return [S.Pose(np.array([1.0, 0.0, 0.0, 0.0]), np.array([x, 0.2, 0.0])) for x in xs]


def test_loop_closure_on_sweeps_against_the_composition(ctxs, fronts):
    """Out and back with spinning sweeps: the loop closes inside the sequence call; loop closure on changes no odometry output; the loop-closure
    oracle driven by the oracle's spin full clouds and the device poses gives the same keyframe schedule, infos and poses_ori bit for bit and
    the same decisions, alignments within the tolerances of test_gpu_loop_closure (against the oracle's alignment of the clouds the device
    aligns), the optimized poses within 1e-8 and the refined clouds bit for bit."""
    from loam_livox_b200 import capi
    from oracle import oracle as O
    from oracle.spin_oracle import SpinExtractor
    import loop_closure_oracle as LCO
    poses = _returning(40) + _returning(40)[1:11]
    raws = [S.make_spinning_scan(16, p, seed=S.SEED + 1600 + k) for k, p in enumerate(poses)]
    a, b = _mapper(ctxs[0], p0=poses[0]), _mapper(ctxs[1], p0=poses[0])
    try:
        c = b.set_loop_closure(**SMALL)
        ra, rb = a.process_new_sweeps(fronts[0][16], raws), b.process_new_sweeps(fronts[1][16], raws)
        assert [entry(*x) for x in ra] == [entry(*x) for x in rb]
        assert a.save() == b.save()
        log, _ = b.loop_log()
        r = b.loop_result()
        kf = [e for e in log if e.kind == capi.LL_LOOP_KEYFRAME]
        al = [e for e in log if e.kind == capi.LL_LOOP_ALIGNMENT]
        cl = [e for e in log if e.kind == capi.LL_LOOP_CLOSED]
        print(f"keyframes {len(kf)}, alignments {[(e.keyframe, e.his, round(e.inlier_threshold, 4), e.decision) for e in al]}, closed {r['closed']}")
        assert r["closed"] and len(cl) == 1 and kf[-1].ending_frame_idx < len(raws)
        assert all(x.status == 1 for x, _ in rb)
        lo = LCO.LoopClosureOracle(c.scans_of_each_keyframe, c.scans_between_two_keyframe,
                                   {k: getattr(c.loop, k) for k, _ in capi.LoopCfg._fields_}, c.map_alignment_inlier_threshold,
                                   dict(line_res=c.map_alignment_resolution, plane_res=c.map_alignment_resolution,
                                        maximum_icp_iteration=c.map_alignment_maximum_icp_iteration,
                                        maximum_residual_block=c.scene_alignment_maximum_residual_block, rng_seed=c.rng_seed, threads=8),
                                   c.surround_pointcloud_resolution, 1.0, 2000, bool(c.incremental_cov), 400, poses[0].q, poses[0].t)
        ex = SpinExtractor(16)
        frozen = []   # each keyframe's line / plane clouds as its analysis left them
        for k, raw in enumerate(raws):
            full = ex.extract(raw)["full"]
            x = rb[k][0]
            lo.step(full, np.array(x.q_w_curr), np.array(x.t_w_curr), k + 1)
            frozen += [(lo.map.cloud(h, capi.LL_CELL_LINE), lo.map.cloud(h, capi.LL_CELL_PLANE)) for h in lo.kfs[len(frozen):]]
            if lo.loop is not None:
                break
        assert [e.ending_frame_idx for e in kf] == lo.ending
        for e, i in zip(kf, lo.infos):
            assert e.info.all_points == i["all_points"]
            assert (e.info.cells, e.info.line_cells, e.info.plane_cells, e.info.accumulate_frames) == (i["cells"], i["line_cells"], i["plane_cells"], i["accumulate_frames"])
            assert np.array(e.info.center, np.float32).tobytes() == i["center"].tobytes()
        assert r["poses_ori"].tobytes() == np.array(lo.poses).tobytes()
        assert [(e.keyframe, e.his, e.decision) for e in al] == [(n, h, d) for n, h, d, _ in lo.decisions]
        # The device aligns against the older keyframe's typed clouds as its analysis left them; the reference (and the composition) extract them
        # from the shared cells at alignment time, which the sweeps since have filled further (DESIGN.md §4.6, deviation (xx)).  So the
        # alignments are held to the tolerances of test_gpu_loop_closure against the oracle's scene alignment of the clouds the device aligns.
        infos = [lo.map.info(h) for h in lo.kfs]
        for e in al:
            t0 = (infos[e.keyframe]["center"] - infos[e.his]["center"]).astype(np.float32).astype(np.float64)
            o, _ = O.scene_align(*frozen[e.keyframe], *frozen[e.his], t_init=t0, accepted_threshold=c.map_alignment_inlier_threshold, **lo.align_kw)
            assert abs(e.inlier_threshold - o.inlier_threshold) <= 1e-3
            assert np.abs(np.array(e.icp_t) - np.array(o.t_w_curr)).max() <= 1e-2
        c0 = cl[0]
        X = lo.optimize((c0.edge.id_begin, c0.edge.id_end), np.concatenate([np.array(c0.edge.q_wxyz), np.array(c0.edge.t)]))
        assert np.abs(X - r["poses_opt"]).max() <= 1e-8
        ref = lo.refined(r["poses_opt"])
        n = len(lo.kfs)
        for k in range(n - 1, -1, -2):
            got = b.loop_cloud(k)
            assert got.shape[0] == ref[k].shape[0] and got[:, :3].tobytes() == ref[k][:, :3].tobytes(), k
    finally:
        a.close(); b.close()


def test_empty_sweeps_with_loop_closure(ctxs):
    """Empty sweeps inside the first keyframe, the first one as the spin handle's first sweep after a larger ll_spin_extract: each hands the
    loop closure an empty cloud, as the reference appends one.  Keyframe schedule, infos and poses equal the loop-closure oracle's bit for bit."""
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_feature
    import loop_closure_oracle as LCO
    from oracle.spin_oracle import SpinExtractor
    raws = vlp(14, S.SEED + 1800)
    empty = np.zeros((0, 4), np.float32)
    stream = [empty] + raws[:2] + [empty] + raws[2:]
    f = Laser_feature(ctxs[1], 16)
    gm = _mapper(ctxs[1])
    try:
        f.extract(S.make_spinning_scan(16, n_azimuth=3600, seed=S.SEED + 1850))   # the handle's device count is now that sweep's
        c = gm.set_loop_closure(**dict(SMALL, loop=dict(SMALL["loop"], minimum_keyframe_differen=100000)))
        out = gm.process_new_sweeps(f, stream)
        assert all(r.status == 1 for r, _ in out)
        log, _ = gm.loop_log()
        assert not [e for e in log if e.kind == capi.LL_LOOP_ERROR]
        kf = [e for e in log if e.kind == capi.LL_LOOP_KEYFRAME]
        lo = LCO.LoopClosureOracle(c.scans_of_each_keyframe, c.scans_between_two_keyframe, {k: getattr(c.loop, k) for k, _ in capi.LoopCfg._fields_},
                                   c.map_alignment_inlier_threshold, {}, c.surround_pointcloud_resolution, 1.0, 2000, bool(c.incremental_cov), 400,
                                   np.array([1.0, 0.0, 0.0, 0.0]), np.zeros(3))
        ex = SpinExtractor(16)
        for k, (raw, (r, _)) in enumerate(zip(stream, out)):
            lo.step(ex.extract(raw)["full"] if raw.shape[0] else empty, np.array(r.q_w_curr), np.array(r.t_w_curr), k + 1)
        assert len(kf) >= 5 and [e.ending_frame_idx for e in kf] == lo.ending
        for e, i in zip(kf, lo.infos):
            assert e.info.all_points == i["all_points"]
            assert (e.info.cells, e.info.line_cells, e.info.plane_cells, e.info.accumulate_frames) == (i["cells"], i["line_cells"], i["plane_cells"], i["accumulate_frames"])
            assert np.array(e.info.center, np.float32).tobytes() == i["center"].tobytes()
        assert gm.loop_result()["poses_ori"].tobytes() == np.array(lo.poses).tobytes()
    finally:
        gm.close(); f.close()


# ---------------------------------------------------------------------------------------------- 9. recovery
def test_recovery_on_a_tracking_stream_changes_nothing(ctxs, fronts):
    raws = vlp(10, S.SEED + 1700)
    ga, gb = _mapper(ctxs[0]), _mapper(ctxs[1])
    try:
        gb.set_recovery()
        assert singles(ga, fronts[0][16], raws[:4]) == singles(gb, fronts[1][16], raws[:4])
        assert seq(ga, fronts[0][16], raws[4:]) == seq(gb, fronts[1][16], raws[4:])
        assert state(ga) == state(gb) and ga.save() == gb.save()
    finally:
        ga.close(); gb.close()
