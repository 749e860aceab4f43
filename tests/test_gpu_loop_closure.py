"""Loop closure inside the streaming mapper (ll_mapper_set_loop_closure, ll_mapper_loop_read / _result / _cloud; DESIGN.md §4.6): it changes no
odometry output through scans, frames and the sequence calls, the sequence calls give the single calls' log and results bit for bit, the
keyframe schedule follows laser_mapping.hpp:1534-1563, a trajectory through the synthetic room that returns to its start closes its loop, work
stops after the loop, and bad configurations are refused with nothing changed."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from loam_livox_b200 import synthetic as S  # noqa: E402

pytestmark = pytest.mark.gpu

N = 24000
STAT_INTS = ("n_corner", "n_surf", "map_corner", "map_surf", "cells_in_fov_corner", "cells_in_fov_surf", "appended_corner", "appended_surf")
# small keyframes and a permissive search, so that a short stream closes keyframes and searches them
SMALL = dict(scans_of_each_keyframe=6, scans_between_two_keyframe=2, reserve_map_points=1 << 21, reserve_history_points=1 << 20, reserve_keyframes=64,
             loop=dict(minimum_keyframe_differen=8, avail_ratio_plane=0.02, avail_ratio_line=0.005), map_alignment_inlier_threshold=0.35)
# the same keyframes without a candidate: no loop closes, so every keyframe of the stream is closed and processed
NOSEARCH = dict(SMALL, loop=dict(SMALL["loop"], minimum_keyframe_differen=100000))


@pytest.fixture(scope="module")
def ctxs():
    from loam_livox_b200.registration import Context
    cs = [Context(0, max_scan_points=60000, max_features=400000) for _ in range(2)]   # max_features: room for the keyframes' typed clouds
    yield cs
    for c in cs:
        c.close()


def _mapper(ctx, mode, p0, pieces=3, **kw):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping
    pipe = capi.PipelineCfg(pieces=pieces, use_piece=0, extractor_leaf_corner=0.1, extractor_leaf_surf=0.2, mapping_leaf_corner=0.1, mapping_leaf_surf=0.4, whole_frame=1)
    st = capi.default_reg_state(mapping_init_accumulate_frames=3, q_w_last=p0.q, t_w_last=p0.t, q_w_curr=p0.q, t_w_curr=p0.t)
    return Laser_mapping(ctx, reg=st, pipeline=pipe, matching_mode=mode, maximum_history_size=400, **kw)


def _b(x):
    return np.array(list(x) if isinstance(x, C.Array) else [x]).tobytes()


def _entry(res):
    from loam_livox_b200 import capi
    return tuple(_b(getattr(res, f)) for f, _ in capi.RegResult._fields_ if not f.startswith("gpu_ms"))


def _stats(st):
    return tuple(getattr(st, f) for f in STAT_INTS)


def _ev(e):
    """an event's bytes without the pose graph's SM clock counters (ll_pg_summary::cycles_*), which time the solve"""
    from loam_livox_b200 import capi
    c = capi.LoopEvent.from_buffer_copy(e)
    c.summary.cycles_eval = c.summary.cycles_elim = c.summary.cycles_border = c.summary.cycles_total = 0
    return bytes(c)


def _returning(n_out=40, step=0.15):
    """Out along the aisle and back to the start."""
    xs = [0.3 + step * k for k in range(n_out)] + [0.3 + step * (n_out - 1 - k) for k in range(n_out)]
    return [S.Pose(np.array([1.0, 0.0, 0.0, 0.0]), np.array([x, 0.2, 0.0])) for x in xs]


def _scans(poses, seed):
    return [S.make_scan(N, p, seed=seed + k) for k, p in enumerate(poses)], [100.0 + 0.1 * k for k in range(len(poses))]


def _expected_schedule(n_steps, each, between):
    """ending frame indices of the keyframes laser_mapping.hpp:1534-1563 closes when every step appends (frame index after step k: k + 1)."""
    open_, ends = [0], []
    for k in range(n_steps):
        open_ = [f + 1 for f in open_]
        if open_[0] >= each:
            ends.append(k + 1)
            open_.pop(0)
        if open_[-1] >= between:
            open_.append(0)
    return ends


# ---------------------------------------------------------------------------------------------- no effect on the odometry
@pytest.mark.parametrize("mode", [0, 1])
def test_loop_closure_changes_no_odometry_scans(ctxs, mode):
    poses = _returning(30)
    raws, stamps = _scans(poses, S.SEED + 5100)
    a, b = _mapper(ctxs[0], mode, poses[0]), _mapper(ctxs[1], mode, poses[0])
    b.set_loop_closure(**NOSEARCH)
    ra = [a.process_new_scan(r, t) for r, t in zip(raws[:20], stamps[:20])] + a.process_new_scans(raws[20:], stamps[20:])
    rb = [b.process_new_scan(r, t) for r, t in zip(raws[:20], stamps[:20])] + b.process_new_scans(raws[20:], stamps[20:])
    assert [_entry(x) for x, _ in ra] == [_entry(x) for x, _ in rb]
    assert [_stats(x) for _, x in ra] == [_stats(x) for _, x in rb]
    qa, ta, fa = a.pose()
    qb, tb, fb = b.pose()
    assert qa.tobytes() == qb.tobytes() and ta.tobytes() == tb.tobytes() and fa == fb
    assert a.save() == b.save()
    log, dropped = b.loop_log()
    from loam_livox_b200 import capi
    kf = [e for e in log if e.kind == capi.LL_LOOP_KEYFRAME]
    assert dropped == 0 and [e.ending_frame_idx for e in kf] == _expected_schedule(len(raws), 6, 2)
    assert all(e.info.cells > 0 and e.info.all_points > 0 for e in kf)
    a.close(); b.close()


@pytest.mark.parametrize("mode", [0, 1])
def test_loop_closure_changes_no_odometry_frames(ctxs, mode):
    poses = _returning(12)
    frames = [S.make_triple_scan(N, p, seed=S.SEED + 5200 + 3 * k) for k, p in enumerate(poses)]
    stamps = [[100.0 + 0.1 * k] * 3 for k in range(len(poses))]
    a, b = _mapper(ctxs[0], mode, poses[0], pieces=2), _mapper(ctxs[1], mode, poses[0], pieces=2)
    b.set_loop_closure(**NOSEARCH)
    ra = [a.process_new_frame(f, s) for f, s in zip(frames[:8], stamps[:8])] + a.process_new_frames(frames[8:], stamps[8:])
    rb = [b.process_new_frame(f, s) for f, s in zip(frames[:8], stamps[:8])] + b.process_new_frames(frames[8:], stamps[8:])
    assert [[_entry(x) for x, _ in f] for f in ra] == [[_entry(x) for x, _ in f] for f in rb]
    assert [[_stats(x) for _, x in f] for f in ra] == [[_stats(x) for _, x in f] for f in rb]
    assert a.save() == b.save()
    log, _ = b.loop_log()
    from loam_livox_b200 import capi
    n_steps = sum(len(f) for f in rb)
    assert [e.ending_frame_idx for e in log if e.kind == capi.LL_LOOP_KEYFRAME] == _expected_schedule(n_steps, 6, 2)
    a.close(); b.close()


# ---------------------------------------------------------------------------------------------- sequence calls = single calls
def _sequence_and_single_calls(ctxs, kind):
    """a: the single calls, b: the sequence call, both with loop closure on; their entries, one per step.  frames: two pieces each, so the
    front ends of the sequence alternate between both arenas while the loop closure reads the full clouds that every front end overwrites."""
    if kind == "scans":
        poses = _returning(20)
        raws, stamps = _scans(poses, S.SEED + 5300)
        a, b = _mapper(ctxs[0], 0, poses[0]), _mapper(ctxs[1], 0, poses[0])
    else:
        poses = _returning(12)
        raws = [S.make_triple_scan(N, p, seed=S.SEED + 5350 + 3 * k) for k, p in enumerate(poses)]
        stamps = [[100.0 + 0.1 * k] * 3 for k in range(len(poses))]
        a, b = _mapper(ctxs[0], 0, poses[0], pieces=2), _mapper(ctxs[1], 0, poses[0], pieces=2)
    for m in (a, b):
        m.set_loop_closure(**SMALL)
    if kind == "scans":
        return a, b, [a.process_new_scan(r, t) for r, t in zip(raws, stamps)], b.process_new_scans(raws, stamps)
    ra = [e for f, s in zip(raws, stamps) for e in a.process_new_frame(f, s)]
    rb = [e for f in b.process_new_frames(raws, stamps) for e in f]
    assert len(ra) == 2 * len(raws)
    return a, b, ra, rb


def test_sequence_calls_give_the_single_calls_log(ctxs):
    for kind in ("scans", "frames"):
        a, b, ra, rb = _sequence_and_single_calls(ctxs, kind)
        assert [_entry(x) for x, _ in ra] == [_entry(x) for x, _ in rb], kind
        la, lb = a.loop_log()[0], b.loop_log()[0]
        assert len(la) > 0 and [_ev(e) for e in la] == [_ev(e) for e in lb], kind
        xa, xb = a.loop_result(), b.loop_result()
        assert xa["closed"] == xb["closed"] and xa["poses_ori"].tobytes() == xb["poses_ori"].tobytes() and xa["poses_opt"].tobytes() == xb["poses_opt"].tobytes(), kind
        a.close(); b.close()


@pytest.mark.parametrize("each,between", [(6, 5), (6, 1), (3, 2)])
def test_schedule_edges(ctxs, each, between):
    from loam_livox_b200 import capi
    poses = _returning(10)
    raws, stamps = _scans(poses, S.SEED + 5400)
    m = _mapper(ctxs[0], 0, poses[0])
    m.set_loop_closure(**dict(NOSEARCH, scans_of_each_keyframe=each, scans_between_two_keyframe=between))
    m.process_new_scans(raws, stamps)
    log, _ = m.loop_log()
    assert [e.ending_frame_idx for e in log if e.kind == capi.LL_LOOP_KEYFRAME] == _expected_schedule(len(raws), each, between)
    r = m.loop_result()
    assert r["poses_ori"].shape[0] == len(_expected_schedule(len(raws), each, between))
    m.close()


# ---------------------------------------------------------------------------------------------- end to end
def test_loop_closes_on_a_returning_trajectory(ctxs):
    poses = _returning(40)
    raws, stamps = _scans(poses, S.SEED + 5500)
    m = _mapper(ctxs[0], 0, poses[0])
    try:
        _returning_trajectory(m, poses, raws, stamps)
    finally:
        m.close()


def _returning_trajectory(m, poses, raws, stamps):
    from loam_livox_b200 import capi
    # keyframe k ends at frame 6 + 2 k: with 36 keyframes between a pair, the first to search is keyframe 35 (x = 0.9 m on the way back)
    # against keyframe 0 (x = 1.05 m), so only the return to the start is searched and the room's 4 m repetition stays out of reach
    m.set_loop_closure(**dict(SMALL, loop=dict(SMALL["loop"], minimum_keyframe_differen=36)))
    m.process_new_scans(raws, stamps)
    log, dropped = m.loop_log()
    r = m.loop_result()
    kf = [e for e in log if e.kind == capi.LL_LOOP_KEYFRAME]
    al = [e for e in log if e.kind == capi.LL_LOOP_ALIGNMENT]
    cl = [e for e in log if e.kind == capi.LL_LOOP_CLOSED]
    print(f"keyframes {len(kf)}, alignments {[(e.keyframe, e.his, round(e.inlier_threshold, 4), e.decision) for e in al]}")
    assert all(e.decision != capi.LL_LOOP_FAILED for e in al)
    assert r["closed"] and len(cl) == 1
    c = cl[0]
    newest, his = c.keyframe, c.his
    # the revisit: a keyframe spans 0.9 m of the path (6 scans), so the two keyframes' paths overlap when their ends are within 1.5 m
    truth = [poses[e.ending_frame_idx - 1] for e in kf]
    assert np.linalg.norm(truth[newest].t - truth[his].t) < 1.5, (newest, his)
    # the edge against the true relative pose (both keyframes face +x: the relative translation is the difference).  The alignment of these
    # 6-scan keyframes scores 0.1995 (a loose fit: the threshold is 0.35) and its edge was measured 0.164 m off the truth on one H100
    rel = truth[his].t - truth[newest].t
    e_edge = np.linalg.norm(np.array(c.edge.t) - rel)
    # the optimized keyframe path is no farther from the truth than the odometry's
    T = np.array([p.t for p in truth])
    e_odo = np.linalg.norm(r["poses_ori"][:, 4:] - T, axis=1).max()
    e_opt = np.linalg.norm(r["poses_opt"][:, 4:] - T, axis=1).max()
    print(f"edge {e_edge:.4f} m off the truth; keyframe path: odometry {e_odo:.4f} m, optimized {e_opt:.4f} m")
    assert e_edge < 0.25
    assert e_opt <= e_odo + 0.02
    # the refined clouds of the published keyframes; the others are refused
    n = r["poses_ori"].shape[0]
    pc = m.loop_cloud(n - 1)
    assert pc.shape[0] > 0 and np.all(pc[:, 3] == 0)
    with pytest.raises(Exception):
        m.loop_cloud(n - 2)
    # no more work after the loop
    more = _scans(_returning(5), S.SEED + 5600)
    m.process_new_scans(more[0], [200.0 + 0.1 * k for k in range(5)])
    assert m.loop_log()[0] == [] and m.loop_result()["poses_ori"].shape[0] == n


# ---------------------------------------------------------------------------------------------- refusals, load
def test_refusals_change_nothing_and_a_loaded_mapper_has_it_off(ctxs):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping
    poses = _returning(8)
    raws, stamps = _scans(poses, S.SEED + 5700)
    m = _mapper(ctxs[0], 0, poses[0])
    m.set_loop_closure(**SMALL)
    m.process_new_scans(raws, stamps)
    before = m.loop_result()
    for bad in (dict(scans_between_two_keyframe=6), dict(scans_between_two_keyframe=7), dict(scans_of_each_keyframe=0),
                dict(map_alignment_resolution=float("nan")), dict(surround_pointcloud_resolution=0.0), dict(incremental_cov=2),
                dict(reserve_keyframes=-1), dict(loop=dict(minimum_similarity_planar=float("inf")))):
        with pytest.raises(Exception):
            m.set_loop_closure(**dict(SMALL, **bad))
        after = m.loop_result()
        assert after["poses_ori"].tobytes() == before["poses_ori"].tobytes()
    img = m.save()
    m2 = Laser_mapping.load(ctxs[1], img)
    r = m2.loop_result()
    assert r["poses_ori"].shape[0] == 0 and not r["closed"] and m2.loop_log()[0] == []
    m2.process_new_scans(raws[:3], [300.0, 300.1, 300.2])
    assert m2.loop_log()[0] == []
    m.set_loop_closure(False)
    assert m.loop_result()["poses_ori"].shape[0] == 0
    with pytest.raises(Exception):
        m.loop_cloud(0)
    m.close(); m2.close()


# ---------------------------------------------------------------------------------------------- parity with the oracle composition
def test_parity_with_the_oracle_composition_and_no_effect_through_the_loop(ctxs):
    """A stream out along the room, back to the start and out again: the loop closes inside the sequence call with steps after it.  Loop closure
    on changes no odometry output; the oracle composition (tests/loop_closure_oracle.py) driven by the device's registration poses gives the same
    keyframe schedule and infos bit for bit, the same candidates and decisions, alignments within the tolerances of
    test_loop_detection_end_to_end_on_the_synthetic_room, the optimized poses on the device's edge within 1e-8, and the refined clouds of the
    published keyframes bit for bit."""
    from loam_livox_b200 import capi
    from oracle import oracle as O
    import loop_closure_oracle as LCO
    poses = _returning(40) + _returning(40)[1:11]
    raws, stamps = _scans(poses, S.SEED + 5800)
    cfg = dict(SMALL, loop=dict(SMALL["loop"], minimum_keyframe_differen=36))
    a, b = _mapper(ctxs[0], 0, poses[0]), _mapper(ctxs[1], 0, poses[0])
    try:
        c = b.set_loop_closure(**cfg)
        ra, rb = a.process_new_scans(raws, stamps), b.process_new_scans(raws, stamps)
        assert [_entry(x) for x, _ in ra] == [_entry(x) for x, _ in rb]
        assert [_stats(x) for _, x in ra] == [_stats(x) for _, x in rb]
        assert a.save() == b.save()
        log, _ = b.loop_log()
        r = b.loop_result()
        assert r["closed"]
        kf = [e for e in log if e.kind == capi.LL_LOOP_KEYFRAME]
        al = [e for e in log if e.kind == capi.LL_LOOP_ALIGNMENT]
        cl = [e for e in log if e.kind == capi.LL_LOOP_CLOSED][0]
        assert kf[-1].ending_frame_idx < len(raws)   # steps ran after the loop closed
        # the composition
        assert all(x.status == 1 for x, _ in rb)   # every step appended
        lo = LCO.LoopClosureOracle(c.scans_of_each_keyframe, c.scans_between_two_keyframe,
                                   {k: getattr(c.loop, k) for k, _ in capi.LoopCfg._fields_}, c.map_alignment_inlier_threshold,
                                   dict(line_res=c.map_alignment_resolution, plane_res=c.map_alignment_resolution,
                                        maximum_icp_iteration=c.map_alignment_maximum_icp_iteration,
                                        maximum_residual_block=c.scene_alignment_maximum_residual_block, rng_seed=c.rng_seed, threads=8),
                                   c.surround_pointcloud_resolution, 1.0, 2000, bool(c.incremental_cov), 400, poses[0].q, poses[0].t)
        ex = O.Extractor()
        for k, (raw, st) in enumerate(zip(raws, stamps)):
            ex.extract(raw, st)
            _, _, full = ex.get_features(0.0, 1.0)
            x = rb[k][0]
            lo.step(full, np.array(x.q_w_curr), np.array(x.t_w_curr), k + 1)
            if lo.loop is not None:
                break
        assert [e.ending_frame_idx for e in kf] == lo.ending
        for e, i in zip(kf, lo.infos):
            assert e.info.all_points == i["all_points"]
            assert (e.info.cells, e.info.line_cells, e.info.plane_cells, e.info.accumulate_frames) == (i["cells"], i["line_cells"], i["plane_cells"], i["accumulate_frames"])
            assert np.array(e.info.center, np.float32).tobytes() == i["center"].tobytes()
            assert (np.float32(e.info.roi_range), np.float32(e.info.ratio_nonzero_line), np.float32(e.info.ratio_nonzero_plane)) == (i["roi_range"], i["ratio_line"], i["ratio_plane"])
        assert r["poses_ori"].tobytes() == np.array(lo.poses).tobytes()
        assert kf[-1].n_candidates == len(lo.last_candidates)
        assert [(e.keyframe, e.his, e.decision) for e in al] == [(n, h, d) for n, h, d, _ in lo.decisions]
        for e, (_, _, _, o) in zip(al, lo.decisions):
            assert abs(e.inlier_threshold - o.inlier_threshold) <= 1e-3
            assert np.abs(np.array(e.icp_t) - np.array(o.t_w_curr)).max() <= 1e-2
        # the optimization on the device's loop edge
        edge = np.concatenate([np.array(cl.edge.q_wxyz), np.array(cl.edge.t)])
        X = lo.optimize((cl.edge.id_begin, cl.edge.id_end), edge)
        assert np.abs(X - r["poses_opt"]).max() <= 1e-8
        # the refined clouds, from the device's optimized poses: every published keyframe, bit for bit
        ref = lo.refined(r["poses_opt"])
        n = len(lo.kfs)
        for k in range(n - 1, -1, -2):
            got = b.loop_cloud(k)
            assert got.shape[0] == ref[k].shape[0] and got[:, :3].tobytes() == ref[k][:, :3].tobytes(), k
    finally:
        a.close(); b.close()

