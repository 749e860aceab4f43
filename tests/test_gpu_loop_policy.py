"""Loops after the first (ll_mapper_set_loop_policy, ll_mapper_loop_edges; DESIGN.md §4.6): the default policy set explicitly is the reference's
single loop bit for bit; a stream that revisits the start twice closes two loops under a multi-loop policy, each edge near the truth and the final
optimized path no worse than the odometry; parity with the loop-closure oracle composition over both loops; no odometry effect through scans
and frames, single and sequence calls; checkpoints between and after the loops continue bit for bit; refusals change nothing."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from loam_livox_b200 import synthetic as S  # noqa: E402
from test_gpu_loop_closure import SMALL, _entry, _ev, _mapper, _returning, _scans, _stats  # noqa: E402

pytestmark = pytest.mark.gpu

# keyframe k ends at frame 6 + 2 k.  With 36 keyframes between a pair the first searched pair is the first return to the start (keyframe 36 on
# the way back against keyframe 0), and the room's 4 m repetition comes within reach only at keyframe 47 (the second pass out at x = 5.4 m
# against keyframe 0 at x = 1.05 m).  Two loops 4 keyframes apart close on the returns to the start before that.
MULTI = dict(SMALL, loop=dict(SMALL["loop"], minimum_keyframe_differen=36))
M, GAP = 2, 4
FIRST_ALIAS = 47


@pytest.fixture(scope="module")
def ctxs():
    from loam_livox_b200.registration import Context
    cs = [Context(0, max_scan_points=60000, max_features=400000) for _ in range(2)]
    yield cs
    for c in cs:
        c.close()


def _stream():
    poses = _returning(40) + _returning(40)[1:]
    raws, stamps = _scans(poses, S.SEED + 6100)
    return poses, raws, stamps


def _kinds(log):
    from loam_livox_b200 import capi
    return ([e for e in log if e.kind == capi.LL_LOOP_KEYFRAME], [e for e in log if e.kind == capi.LL_LOOP_ALIGNMENT],
            [e for e in log if e.kind == capi.LL_LOOP_CLOSED])


def _published(m, n_opt):
    return {k: m.loop_cloud(k) for k in range(n_opt - 1, -1, -2)}


@pytest.fixture(scope="module")
def two_loops(ctxs):
    """The two-revisit stream through one sequence call under the multi-loop policy: its results, log, edges and published clouds."""
    poses, raws, stamps = _stream()
    m = _mapper(ctxs[0], 0, poses[0])
    try:
        cfg = m.set_loop_closure(**MULTI)
        m.set_loop_policy(M, GAP)
        out = m.process_new_scans(raws, stamps)
        log, dropped = m.loop_log()
        r = m.loop_result()
        edges = m.loop_edges()
        n_opt = max(edges[-1].id_begin, edges[-1].id_end) + 1 if edges else 0
        clouds = _published(m, n_opt) if edges else {}
        image = m.save_loop()
    finally:
        m.close()
    return dict(poses=poses, raws=raws, stamps=stamps, cfg=cfg, out=out, log=log, dropped=dropped, r=r, edges=edges, n_opt=n_opt, clouds=clouds,
                image=image)


# ---------------------------------------------------------------------------------------------- the default policy is the reference
def test_the_default_policy_set_explicitly_changes_nothing(ctxs):
    from loam_livox_b200 import capi
    poses = _returning(40) + _returning(40)[1:11]
    raws, stamps = _scans(poses, S.SEED + 5800)
    a, b = _mapper(ctxs[0], 0, poses[0]), _mapper(ctxs[1], 0, poses[0])
    try:
        a.set_loop_closure(**MULTI)
        b.set_loop_closure(**MULTI)
        p = b.set_loop_policy()
        assert (p.max_loops, p.min_keyframes_between_loops) == (1, 0)
        ra, rb = a.process_new_scans(raws, stamps), b.process_new_scans(raws, stamps)
        assert [_entry(x) for x, _ in ra] == [_entry(x) for x, _ in rb]
        la, lb = a.loop_log()[0], b.loop_log()[0]
        assert len(_kinds(la)[2]) == 1 and [_ev(e) for e in la] == [_ev(e) for e in lb]
        xa, xb = a.loop_result(), b.loop_result()
        assert xa["closed"] and xb["closed"]
        assert xa["poses_ori"].tobytes() == xb["poses_ori"].tobytes() and xa["poses_opt"].tobytes() == xb["poses_opt"].tobytes()
        assert bytes(xa["edge"]) == bytes(xb["edge"])
        ea, eb = a.loop_edges(), b.loop_edges()
        assert len(ea) == 1 and bytes(ea[0]) == bytes(eb[0]) == bytes(xa["edge"])
        n = xa["poses_ori"].shape[0]
        for k, c in _published(a, n).items():
            assert c.tobytes() == b.loop_cloud(k).tobytes(), k
        ia, ib = a.save_loop(), b.save_loop()
        assert ia == ib and int.from_bytes(ia[8:12], "little") == capi.LL_LOOP_IMAGE_VERSION
    finally:
        a.close(); b.close()


# ---------------------------------------------------------------------------------------------- two revisits, two loops
def test_two_revisits_close_two_loops(two_loops):
    from loam_livox_b200 import capi
    T = two_loops
    log, r, edges, poses = T["log"], T["r"], T["edges"], T["poses"]
    kf, al, cl = _kinds(log)
    print(f"keyframes {len(kf)}, alignments {[(e.keyframe, e.his, round(e.inlier_threshold, 4), e.decision) for e in al]}")
    print(f"loops (newest, his): {[(e.keyframe, e.his) for e in cl]}; the room's repetition first reachable at keyframe {FIRST_ALIAS}")
    assert T["dropped"] == 0 and all(e.decision != capi.LL_LOOP_FAILED for e in al)
    assert 2 <= len(cl) <= M and r["closed"]
    newest = [e.keyframe for e in cl]
    assert all(b - a >= GAP for a, b in zip(newest, newest[1:])), newest
    assert newest[-1] < FIRST_ALIAS
    # keyframes inside the gap are recorded, not searched
    for e in kf:
        last = [x for x in newest if x < e.keyframe]
        if last and e.keyframe - last[-1] < GAP:
            assert e.n_candidates == 0 and not [a for a in al if a.keyframe == e.keyframe], e.keyframe
    # no event after the M-th loop, and no keyframe after its closing one
    if len(cl) == M:
        assert log[-1].kind == capi.LL_LOOP_CLOSED and kf[-1].keyframe == newest[-1]
    # the edges: in closing order, as the events have them, each near the true relative pose of a true revisit
    assert [bytes(e) for e in edges] == [bytes(e.edge) for e in cl]
    truth = [poses[e.ending_frame_idx - 1] for e in kf]
    for e in cl:
        d_pair = np.linalg.norm(truth[e.keyframe].t - truth[e.his].t)
        e_edge = np.linalg.norm(np.array(e.edge.t) - (truth[e.his].t - truth[e.keyframe].t))
        print(f"loop {e.keyframe} -> {e.his}: true positions {d_pair:.3f} m apart, edge {e_edge:.4f} m off the truth")
        assert d_pair < 1.5 and e_edge < 0.25
    Tt = np.array([p.t for p in truth])
    e_odo = np.linalg.norm(r["poses_ori"][:, 4:] - Tt, axis=1).max()
    e_opt = np.linalg.norm(r["poses_opt"][:, 4:] - Tt, axis=1).max()
    print(f"keyframe path: odometry {e_odo:.4f} m, optimized over {len(cl)} loops {e_opt:.4f} m")
    assert e_opt <= e_odo + 0.02
    assert T["n_opt"] == newest[-1] + 1 and all(c.shape[0] > 0 and np.all(c[:, 3] == 0) for c in T["clouds"].values())
    assert int.from_bytes(T["image"][8:12], "little") == capi.LL_LOOP_IMAGE_VERSION_POLICY


# ---------------------------------------------------------------------------------------------- parity with the oracle composition
def test_parity_with_the_oracle_composition_over_both_loops(two_loops):
    from loam_livox_b200 import capi
    from oracle import oracle as O
    import loop_policy_oracle as LPO
    T = two_loops
    c, rb, log, r = T["cfg"], T["out"], T["log"], T["r"]
    kf, al, cl = _kinds(log)
    assert all(x.status == 1 for x, _ in rb)
    lo = LPO.LoopPolicyOracle(c.scans_of_each_keyframe, c.scans_between_two_keyframe, {k: getattr(c.loop, k) for k, _ in capi.LoopCfg._fields_},
                               c.map_alignment_inlier_threshold,
                               dict(line_res=c.map_alignment_resolution, plane_res=c.map_alignment_resolution,
                                    maximum_icp_iteration=c.map_alignment_maximum_icp_iteration,
                                    maximum_residual_block=c.scene_alignment_maximum_residual_block, rng_seed=c.rng_seed, threads=8),
                               c.surround_pointcloud_resolution, 1.0, 2000, bool(c.incremental_cov), 400, T["poses"][0].q, T["poses"][0].t,
                               max_loops=M, min_keyframes_between_loops=GAP)
    ex = O.Extractor()
    for k, (raw, st) in enumerate(zip(T["raws"], T["stamps"])):
        ex.extract(raw, st)
        _, _, full = ex.get_features(0.0, 1.0)
        x = rb[k][0]
        lo.step(full, np.array(x.q_w_curr), np.array(x.t_w_curr), k + 1)
        if LPO.loops_done(len(lo.loops), M):
            break
    assert [e.ending_frame_idx for e in kf] == lo.ending
    for e, i in zip(kf, lo.infos):
        assert e.info.all_points == i["all_points"]
        assert (e.info.cells, e.info.line_cells, e.info.plane_cells, e.info.accumulate_frames) == (i["cells"], i["line_cells"], i["plane_cells"], i["accumulate_frames"])
        assert np.array(e.info.center, np.float32).tobytes() == i["center"].tobytes()
        assert (np.float32(e.info.roi_range), np.float32(e.info.ratio_nonzero_line), np.float32(e.info.ratio_nonzero_plane)) == (i["roi_range"], i["ratio_line"], i["ratio_plane"])
    assert r["poses_ori"].tobytes() == np.array(lo.poses).tobytes()
    assert [e.n_candidates for e in kf] == lo.n_candidates
    assert [(e.keyframe, e.his, e.decision) for e in al] == [(n, h, d) for n, h, d, _ in lo.decisions]
    assert [(e.keyframe, e.his) for e in cl] == [(n, h) for n, h, _ in lo.loops]
    for e, (_, _, _, o) in zip(al, lo.decisions):
        assert abs(e.inlier_threshold - o.inlier_threshold) <= 1e-3
        assert np.abs(np.array(e.icp_t) - np.array(o.t_w_curr)).max() <= 1e-2
    # the optimization over every loop edge the device built, from the odometry poses
    n_opt = T["n_opt"]
    X = lo.optimize_loops([((e.id_begin, e.id_end), np.concatenate([np.array(e.q_wxyz), np.array(e.t)])) for e in T["edges"]])
    print(f"optimized poses: {np.abs(X - r['poses_opt'][:n_opt]).max():.2e} from the oracle's over {len(T['edges'])} loop edges")
    assert np.abs(X - r["poses_opt"][:n_opt]).max() <= 1e-8
    ref = lo.refined_upto(r["poses_opt"], n_opt)
    for k, got in T["clouds"].items():
        assert got.shape[0] == ref[k].shape[0] and got[:, :3].tobytes() == ref[k][:, :3].tobytes(), k


# ---------------------------------------------------------------------------------------------- no effect on the odometry
@pytest.mark.parametrize("mode", [0, 1])
def test_no_odometry_effect_and_sequence_calls_give_the_single_calls_log_scans(ctxs, mode):
    poses, raws, stamps = _stream()
    # one mapper per context at a time (a mapper resets its context's extractor bookkeeping): a, then c on the first context
    a = _mapper(ctxs[0], mode, poses[0])
    try:
        ra = a.process_new_scans(raws, stamps)
        qa, ta, fa = a.pose()
        ia = a.save()
    finally:
        a.close()
    b, c = _mapper(ctxs[1], mode, poses[0]), _mapper(ctxs[0], mode, poses[0])
    try:
        for m in (b, c):
            m.set_loop_closure(**MULTI)
            m.set_loop_policy(M, GAP)
        rb = b.process_new_scans(raws, stamps)
        rc = [c.process_new_scan(x, t) for x, t in zip(raws, stamps)]
        assert [_entry(x) for x, _ in ra] == [_entry(x) for x, _ in rb] == [_entry(x) for x, _ in rc]
        assert [_stats(x) for _, x in ra] == [_stats(x) for _, x in rb] == [_stats(x) for _, x in rc]
        qb, tb, fb = b.pose()
        assert qa.tobytes() == qb.tobytes() and ta.tobytes() == tb.tobytes() and fa == fb
        assert ia == b.save() == c.save()
        lb, lc = b.loop_log()[0], c.loop_log()[0]
        print(f"mode {mode}: {len(_kinds(lb)[2])} loops")
        assert [_ev(e) for e in lb] == [_ev(e) for e in lc]
        xb, xc = b.loop_result(), c.loop_result()
        assert xb["poses_ori"].tobytes() == xc["poses_ori"].tobytes() and xb["poses_opt"].tobytes() == xc["poses_opt"].tobytes()
        assert [bytes(e) for e in b.loop_edges()] == [bytes(e) for e in c.loop_edges()]
        assert b.save_loop() == c.save_loop()
    finally:
        b.close(); c.close()


@pytest.mark.parametrize("mode", [0, 1])
def test_no_odometry_effect_and_sequence_calls_give_the_single_calls_log_frames(ctxs, mode):
    poses = _returning(12)
    frames = [S.make_triple_scan(24000, p, seed=S.SEED + 6200 + 3 * k) for k, p in enumerate(poses)]
    stamps = [[100.0 + 0.1 * k] * 3 for k in range(len(poses))]
    a = _mapper(ctxs[0], mode, poses[0], pieces=2)
    try:
        ra = a.process_new_frames(frames, stamps)
        ia = a.save()
    finally:
        a.close()
    b, c = _mapper(ctxs[1], mode, poses[0], pieces=2), _mapper(ctxs[0], mode, poses[0], pieces=2)
    try:
        for m in (b, c):   # a permissive search, so that several loops close (aliases included: only the equality matters here)
            m.set_loop_closure(**SMALL)
            m.set_loop_policy(3, 2)
        rb = b.process_new_frames(frames, stamps)
        rc = [c.process_new_frame(f, s) for f, s in zip(frames, stamps)]
        assert [[_entry(x) for x, _ in f] for f in ra] == [[_entry(x) for x, _ in f] for f in rb] == [[_entry(x) for x, _ in f] for f in rc]
        assert [[_stats(x) for _, x in f] for f in ra] == [[_stats(x) for _, x in f] for f in rb] == [[_stats(x) for _, x in f] for f in rc]
        assert ia == b.save() == c.save()
        lb, lc = b.loop_log()[0], c.loop_log()[0]
        print(f"mode {mode}: {len(_kinds(lb)[2])} loops")
        assert len(lb) > 0 and [_ev(e) for e in lb] == [_ev(e) for e in lc]
        xb, xc = b.loop_result(), c.loop_result()
        assert xb["poses_ori"].tobytes() == xc["poses_ori"].tobytes() and xb["poses_opt"].tobytes() == xc["poses_opt"].tobytes()
        assert [bytes(e) for e in b.loop_edges()] == [bytes(e) for e in c.loop_edges()]
    finally:
        b.close(); c.close()


# ---------------------------------------------------------------------------------------------- checkpoints between and after the loops
def test_checkpoints_between_and_after_the_loops_continue_bit_for_bit(ctxs, two_loops):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import Laser_mapping
    T = two_loops
    poses, raws, stamps = T["poses"], T["raws"], T["stamps"]
    kf, _, cl = _kinds(T["log"])
    assert len(cl) >= 2
    end = {e.keyframe: e.ending_frame_idx for e in kf}
    s1, s2 = end[cl[0].keyframe] + 3, end[cl[1].keyframe] + 3
    assert s1 < end[cl[1].keyframe] and s2 <= len(raws)
    more, more_st = _scans(_returning(5), S.SEED + 6300)[0], [300.0 + 0.1 * k for k in range(5)]
    a = _mapper(ctxs[0], 0, poses[0])
    held = []
    try:
        a.set_loop_closure(**MULTI)
        a.set_loop_policy(M, GAP)
        a.process_new_scans(raws[:s1], stamps[:s1])
        # between the loops: the latest optimization covers n_opt keyframes, the later ones keep their odometry poses and publish nothing
        r = a.loop_result()
        n_opt, K = cl[0].keyframe + 1, r["poses_ori"].shape[0]
        assert r["closed"] and K > n_opt and r["poses_opt"][n_opt:].tobytes() == r["poses_ori"][n_opt:].tobytes()
        assert len(a.loop_edges()) == 1 and a.loop_cloud(n_opt - 1).shape[0] > 0
        for k in (K - 1, n_opt - 2):
            with pytest.raises(Exception):
                a.loop_cloud(k)
        m1, l1 = a.save(), a.save_loop()
        assert int.from_bytes(l1[8:12], "little") == capi.LL_LOOP_IMAGE_VERSION_POLICY
        # a policy after a loop is refused and changes nothing
        with pytest.raises(Exception):
            a.set_loop_policy(3, 0)
        with pytest.raises(Exception):
            a.set_loop_policy()
        assert a.save_loop() == l1
        b = Laser_mapping.load(ctxs[1], m1)
        held.append(b)
        b.load_loop(l1)
        assert b.save_loop() == l1
        for m in (a, b):
            m.process_new_scans(raws[s1:s2], stamps[s1:s2])
        m2, l2 = a.save(), a.save_loop()
        assert b.save_loop() == l2
        c = Laser_mapping.load(ctxs[1], m2)
        held.append(c)
        c.load_loop(l2)
        assert c.save_loop() == l2
        for m in (a, b, c):
            m.process_new_scans(raws[s2:], stamps[s2:])
            m.process_new_scans(more, more_st)
        logs = [[_ev(e) for e in m.loop_log()[0]] for m in (a, b, c)]
        assert logs[0] == logs[1] == logs[2] and logs[0] == [_ev(e) for e in T["log"]]
        res = [m.loop_result() for m in (a, b, c)]
        for x in res[1:]:
            assert x["closed"] == res[0]["closed"] and bytes(x["edge"]) == bytes(res[0]["edge"])
            assert x["poses_ori"].tobytes() == res[0]["poses_ori"].tobytes() and x["poses_opt"].tobytes() == res[0]["poses_opt"].tobytes()
        edges = [[bytes(e) for e in m.loop_edges()] for m in (a, b, c)]
        assert edges[0] == edges[1] == edges[2] == [bytes(e) for e in T["edges"]]
        for k, ref in T["clouds"].items():
            for m in (a, b, c):
                assert m.loop_cloud(k).tobytes() == ref.tobytes(), k
        imgs = [m.save_loop() for m in (a, b, c)]
        assert imgs[0] == imgs[1] == imgs[2]
    finally:
        a.close()
        for m in held:
            m.close()


# ---------------------------------------------------------------------------------------------- refusals
def test_refusals_change_nothing(ctxs):
    from loam_livox_b200 import capi
    poses = _returning(8)
    raws, stamps = _scans(poses, S.SEED + 6400)
    m = _mapper(ctxs[0], 0, poses[0])
    try:
        with pytest.raises(Exception):
            m.set_loop_policy(2, 0)   # loop closure off
        m.set_loop_closure(**MULTI)
        m.process_new_scans(raws[:8], stamps[:8])
        log = m.loop_log()[0]   # (drained first: the loop image holds the unread events)
        before = m.save_loop()
        for bad in (dict(max_loops=0), dict(max_loops=capi.LL_MAX_LOOPS + 1), dict(max_loops=2, min_keyframes_between_loops=-1)):
            with pytest.raises(Exception):
                m.set_loop_policy(**bad)
            assert m.save_loop() == before, bad
        assert int.from_bytes(before[8:12], "little") == capi.LL_LOOP_IMAGE_VERSION
        m.set_loop_policy(capi.LL_MAX_LOOPS, 3)
        assert int.from_bytes(m.save_loop()[8:12], "little") == capi.LL_LOOP_IMAGE_VERSION_POLICY
        m.set_loop_policy()
        assert m.save_loop() == before
        m.set_loop_policy(4, 1)
        m.set_loop_closure(**MULTI)   # resets the policy
        assert int.from_bytes(m.save_loop()[8:12], "little") == capi.LL_LOOP_IMAGE_VERSION
        assert log and m.loop_edges() == []
    finally:
        m.close()
