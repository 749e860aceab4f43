"""Keyframes over a full-resolution cell map (ll_keyframe_append / ll_keyframe_analyze) and the loop candidate search (ll_loop_search) on the
device, against the keyframe oracle (oracle/orc_keyframe.hpp)."""
import numpy as np
import pytest

import keyframe_reference as K
from loam_livox_b200 import capi
from loam_livox_b200.registration import Context, Keyframe, Points_cloud_map, loop_search

pytestmark = pytest.mark.gpu


def _scene(seed, n=30000, shift=(0.0, 0.0)):
    """A room corner: floor, two walls and poles, moved by `shift`, with a little noise."""
    r = np.random.default_rng(seed)
    sx, sy = shift
    parts = [np.c_[r.uniform(0, 8, n), r.uniform(0, 6, n), r.normal(0, 0.01, n)],
             np.c_[r.normal(0, 0.01, n // 2), r.uniform(0, 6, n // 2), r.uniform(0, 3, n // 2)],
             np.c_[r.uniform(0, 8, n // 2), r.normal(6, 0.01, n // 2), r.uniform(0, 3, n // 2)]]
    for px in (2.1, 4.3, 6.2):
        parts.append(np.c_[r.normal(px, 0.01, n // 10), r.normal(3.1, 0.01, n // 10), r.uniform(0, 3, n // 10)])
    p = np.vstack(parts)
    p[:, 0] += sx
    p[:, 1] += sy
    return np.c_[p, np.zeros(len(p))].astype(np.float32)


def _pair(ctx, revisit=2147483647, incremental=False):
    return Points_cloud_map(ctx, 1.0, revisit, 0), K.OracleMap(1.0, revisit, incremental)


def _check_keyframe(ctx, g, kf, o, ko, incremental):
    info = kf.analyze(g, incremental)
    o.analyze(ko)
    oi = o.info(ko)
    keys, inc, typ, vec = kf.cells()
    okeys, oinc, otyp, ovec = o.cells(ko)
    assert np.array_equal(keys, okeys) and np.array_equal(inc, oinc)
    # the device types in the oracle's arithmetic (float covariance, fp64 Jacobi): no disagreement is expected, so none is allowed
    assert int((typ != otyp).sum()) == 0
    assert np.array_equal(vec, ovec)
    assert (info.cells, info.line_cells, info.plane_cells, info.accumulate_frames) == (oi["cells"], oi["line_cells"], oi["plane_cells"],
                                                                                     oi["accumulate_frames"])
    assert np.array_equal(np.array(info.center, np.float32), oi["center"]) and np.float32(info.roi_range) == oi["roi_range"]
    assert np.float32(info.ratio_nonzero_line) == oi["ratio_line"] and np.float32(info.ratio_nonzero_plane) == oi["ratio_plane"]
    imgs, oimgs = kf.images(), o.images(ko)
    assert np.array_equal(imgs[:2], oimgs[:2])   # integer counts
    assert np.abs(imgs[2:] - oimgs[2:]).max() <= 1e-6 * max(1.0, float(oimgs[:2].max()))
    for which in (capi.LL_CELL_LINE, capi.LL_CELL_PLANE, capi.LL_CELL_ALL):
        assert np.array_equal(kf.extract_specify_points(which), o.cloud(ko, which))
    return info


def test_append_leaves_the_map_as_cellmap_append_and_cell_sets_equal_the_oracle(ctx):
    plain = Points_cloud_map(ctx, 1.0, 3, 0)
    g, o = _pair(ctx, 3)
    kfs = [Keyframe(ctx) for _ in range(3)]
    oks = [o.new_keyframe() for _ in range(3)]
    base = np.array([[0.1, 0.1, 0.1, 0]], np.float32)
    clouds = [np.vstack([base, base + [1, 0, 0, 0]]),                                                        # first append: every touched cell
              np.vstack([base + [2, 0, 0, 0]] * 2 + [base + [3, 0, 0, 0]] * 3 + [base + [4, 0, 0, 0]] * 4),   # 2 / 3 / 4 points
              _scene(1, 5000), _scene(2, 5000), np.vstack([base] * 3), _scene(3, 5000), np.vstack([base] * 5), _scene(4, 4000)]
    opens = [[0], [0, 1], [0, 1], [1, 2], [0, 1, 2], [2], [0, 2], [1]]
    for c, op in zip(clouds, opens):
        plain.append_cloud(c)
        Keyframe.append(ctx, g, c, [kfs[i] for i in op])
        o.append(c, [oks[i] for i in op])
        assert plain.stats() == g.stats()
        assert g.stats()[0] == o.cell_count()
        for kf, ko in zip(kfs, oks):
            k, e, _, _ = kf.cells(analyzed=False)
            ok, oe, _, _ = o.cells(ko)
            assert np.array_equal(k, ok) and np.array_equal(e, oe)
    q, t = np.array([1.0, 0, 0, 0]), np.array([4.0, 3.0, 1.0])
    a, na = plain.assemble(q, t, 100.0, 180.0, 0.1, replace=False)
    b, nb = g.assemble(q, t, 100.0, 180.0, 0.1, replace=False)
    assert na == nb and np.array_equal(a, b)
    assert kfs[1].cells(analyzed=False)[1].max() >= 1   # a revisited cell's new incarnation


@pytest.mark.parametrize("incremental", [False, True])
def test_analyze_equals_the_oracle(ctx, incremental):
    g, o = _pair(ctx, 4, incremental)
    kfs = [Keyframe(ctx) for _ in range(2)]
    oks = [o.new_keyframe() for _ in range(2)]
    for s in range(6):
        c = _scene(10 + s, 8000, shift=(0.05 * s, 0.02 * s))
        op = [0] if s < 3 else [0, 1]
        Keyframe.append(ctx, g, c, [kfs[i] for i in op])
        o.append(c, [oks[i] for i in op])
    for kf, ko in zip(kfs, oks):
        info = _check_keyframe(ctx, g, kf, o, ko, incremental)
        assert info.line_cells > 0 and info.plane_cells > 0


def test_keyframe_without_line_cells_and_empty_keyframe(ctx):
    g, o = _pair(ctx)
    kf, ko = Keyframe(ctx), o.new_keyframe()
    r = np.random.default_rng(3)
    floor = np.c_[r.uniform(0, 6, 20000), r.uniform(0, 6, 20000), r.normal(0, 0.01, 20000), np.zeros(20000)].astype(np.float32)
    Keyframe.append(ctx, g, floor, [kf])
    o.append(floor, [ko])
    info = _check_keyframe(ctx, g, kf, o, ko, False)
    assert info.line_cells == 0 and info.ratio_nonzero_line == 0.0
    dev, n = kf.device_cloud(capi.LL_CELL_PLANE)
    assert dev and n == info.plane_points > 0
    empty = Keyframe(ctx)
    info = empty.analyze(g)
    assert info.cells == 0 and info.roi_range == 0.0 and not empty.images().any()


def _keyframes(ctx, n, per=3000, seed=0):
    """n keyframes, one scan each, along a path that comes back to its start."""
    g, o = _pair(ctx)
    kfs, oks = [], []
    for k in range(n):
        ang = 2 * np.pi * k / n
        c = _scene(seed + k, per, shift=(3 * np.cos(ang), 3 * np.sin(ang)))
        kf, ko = Keyframe(ctx), o.new_keyframe()
        Keyframe.append(ctx, g, c, [kf])
        o.append(c, [ko])
        kf.analyze(g)
        o.analyze(ko)
        kfs.append(kf)
        oks.append(ko)
    return g, o, kfs, oks


@pytest.mark.parametrize("n", [2, 40, 300])
def test_search_equals_the_oracle(ctx, n):
    g, o, kfs, oks = _keyframes(ctx, n, per=1500 if n > 100 else 3000)
    infos = [kf.info() for kf in kfs]
    cells = np.array([i.cells for i in infos], np.int64)
    roi = np.array([i.roi_range for i in infos], np.float32)
    rp = np.array([i.ratio_nonzero_plane for i in infos], np.float32)
    rl = np.array([i.ratio_nonzero_line for i in infos], np.float32)
    imgs = np.stack([np.stack([o.images(k)[3], o.images(k)[2]]) for k in oks])
    newest = n - 1
    osims, ocand = K.oracle_search(cells, roi, rp, rl, imgs, newest)
    for cfg in (K.DEFAULT_CFG, dict(K.DEFAULT_CFG, minimum_keyframe_differen=1, minimum_similarity_planar=0.5, plane_with_line=0.3,
                                     minimum_similarity_linear=0.3)):
        sp, sl, cand = loop_search(ctx, kfs, newest, capi.default_loop_cfg(**cfg))
        # the device sums in the oracle's order: the similarities are bit for bit
        assert np.array_equal(sp, osims[:, 0]) and np.array_equal(sl, osims[:, 1])
        assert cand == K.oracle_gates(cells, roi, rp, rl, osims, newest, cfg) == K.numpy_gates(cells, roi, rp, rl, np.c_[sp, sl], newest, cfg)
    assert ocand == K.oracle_gates(cells, roi, rp, rl, osims, newest)


def test_search_is_deterministic_across_runs_and_contexts(ctx):
    _, _, kfs, _ = _keyframes(ctx, 12, seed=50)
    a = loop_search(ctx, kfs, cfg=capi.default_loop_cfg(minimum_keyframe_differen=1))
    b = loop_search(ctx, kfs, cfg=capi.default_loop_cfg(minimum_keyframe_differen=1))
    ctx2 = Context(0, max_scan_points=20000, max_features=20000)
    try:
        _, _, kfs2, _ = _keyframes(ctx2, 12, seed=50)
        c = loop_search(ctx2, kfs2, cfg=capi.default_loop_cfg(minimum_keyframe_differen=1))
        for k in range(12):
            assert np.array_equal(kfs[k].images(), kfs2[k].images())
        for x, y in ((a, b), (a, c)):
            assert np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) and x[2] == y[2]
        for kf in kfs2:
            kf.close()
    finally:
        ctx2.close()


def test_loop_detection_end_to_end_on_the_synthetic_room(ctx):
    """The reference's loop closure from the full clouds on (laser_mapping.hpp:919-1089, 1524-1533): a drifted trajectory through the synthetic
    room that comes back to its start; keyframes of two scans each through ll_keyframe_append; every closed keyframe analyzed and searched; the
    caller's loop of INTEGRATION.md over the candidates (his ascending, ll_scene_align on the device-resident typed clouds with t_init from the
    two centres, `his += 10` after a score over twice the threshold, stop at the first true loop); the loop edge and the pose graph.  The oracle
    runs the same flow: same candidates and decisions, alignments and loop edge within 1 cm, optimized poses within 3 cm, and its error falls too."""
    from oracle import oracle as O
    import pose_graph_reference as R
    from loam_livox_b200 import synthetic as S
    from loam_livox_b200.registration import PoseGraph, Scene_alignment, pg_edges, pg_loop_edge
    from test_gpu_pose_graph import _comp, _inv, _move
    rng = np.random.default_rng(90)
    room = np.vstack(S.make_map(20000, 200000, seed=S.SEED + 90))
    xs = [2.0, 9.0, 16.0, 23.0, 30.0, 2.4]   # out along the room, then back at the start
    n = len(xs)
    truth = np.zeros((n, 7))
    truth[:, 0] = 1.0
    truth[:, 4] = xs
    truth[:, 5] = 0.3 * np.sin(np.arange(n))
    X, ids, meas = R.chain_graph(truth, rng, (), dt=0.04, da=0.004)
    before = np.linalg.norm(X[-1, 4:] - truth[-1, 4:])
    assert 0.05 < before < 0.5
    # a room of a few plane directions: its images fill fewer pixels than the 300-scan keyframes avail_ratio_* (:894-895) were set for.  The room
    # repeats every 4 m (the pillar pitch): views 20-28 m apart align onto each other as well as the revisit does (the oracle scores 0.18-0.20
    # for both), so the keyframe difference lets only the last keyframe search; thr = map_alignment_inlier_threshold's default 0.35 (:703).
    thr, cfg = 0.35, dict(K.DEFAULT_CFG, minimum_keyframe_differen=n, avail_ratio_plane=0.02, avail_ratio_line=0.005)
    # the first keyframe sees less than the last one: the cell-count line (:1030) passes a pair only when the newest has at least as many cells
    radius = [5.0] + [7.5] * (n - 2) + [9.5]
    g, o = _pair(ctx, revisit=4)
    sa = Scene_alignment(ctx, accepted_threshold=thr)   # m_scene_align.m_accepted_threshold = the loop threshold (:897)
    kfs, oks, decided, loop = [], [], [], None
    for k in range(n):
        near = room[np.linalg.norm(room[:, :2] - truth[k, 4:6], axis=1) < radius[k]]
        D = _comp(X[k], _inv(truth[k]))   # the drifted map holds keyframe k's points at X_k T_k^-1 of the room
        kf, ko = Keyframe(ctx), o.new_keyframe()
        for half in (near[0::2], near[1::2]):
            c = _move(half, D)
            Keyframe.append(ctx, g, c, [kf])
            o.append(c, [ko])
        kf.analyze(g)
        o.analyze(ko)
        kfs.append(kf)
        oks.append(ko)
        newest = k
        if newest == 0:
            continue
        sp, sl, cand = loop_search(ctx, kfs, newest, capi.default_loop_cfg(**cfg))
        infos = [x.info() for x in kfs]
        imgs = np.stack([np.stack([o.images(j)[3], o.images(j)[2]]) for j in oks])
        osims, ocand = K.oracle_search(np.array([i.cells for i in infos], np.int64), np.array([i.roi_range for i in infos], np.float32),
                                       np.array([i.ratio_nonzero_plane for i in infos], np.float32),
                                       np.array([i.ratio_nonzero_line for i in infos], np.float32), imgs, newest, cfg)
        assert cand == ocand and np.array_equal(sp, osims[:, 0]) and np.array_equal(sl, osims[:, 1])
        skip_to = -1
        for his in cand:
            if his <= skip_to:
                continue
            r = sa.align_keyframes(kfs[newest], kfs[his])
            t0 = (o.info(newest)["center"] - o.info(his)["center"]).astype(np.float32).astype(np.float64)
            ores, _ = O.scene_align(o.cloud(newest, capi.LL_CELL_LINE), o.cloud(newest, capi.LL_CELL_PLANE), o.cloud(his, capi.LL_CELL_LINE),
                                    o.cloud(his, capi.LL_CELL_PLANE), t_init=t0, accepted_threshold=thr, threads=8)
            # these typed clouds are ~10x the residual-block cap (5000): device and oracle alignments differ by a few mm and mrad here
            assert abs(r.inlier_threshold - ores.inlier_threshold) <= 1e-3
            assert np.abs(np.array(r.t_w_curr) - np.array(ores.t_w_curr)).max() <= 1e-2
            decided.append((newest, his, r.inlier_threshold))
            if r.inlier_threshold > 2 * thr:
                skip_to = his + 10
                continue
            if r.inlier_threshold < thr:
                loop = (newest, his, np.concatenate([np.array(r.q_w_curr), np.array(r.t_w_curr)]),
                        np.concatenate([np.array(ores.q_w_curr), np.array(ores.t_w_curr)]))
                break
        if loop:
            break
    # detection: the revisit of the start is found and is the loop
    assert loop is not None and (loop[0], loop[1]) == (n - 1, 0), decided
    b, a, K_dev, K_orc = loop
    e = pg_loop_edge(K_dev[:4], K_dev[4:], X[a], a, X[b], b)
    (ob, oa), om = R.oracle_loop_edge(K_orc[:4], K_orc[4:], X[a], a, X[b], b)
    em = np.concatenate([np.array(e.q_wxyz), np.array(e.t)])
    assert (e.id_begin, e.id_end) == (ob, oa) == (b, a) and np.abs(em - om).max() < 1e-2
    ids2 = np.concatenate([ids, [[b, a]]]).astype(np.int32)
    pg = PoseGraph(ctx, 64, 64)
    xd, _ = pg.optimize(X, pg_edges(ids2[:, 0], ids2[:, 1], np.concatenate([meas, [em]])[:, :4], np.concatenate([meas, [em]])[:, 4:]))
    pg.close()
    assert np.abs(xd[:, 4:] - R.oracle_optimize(X, ids2, np.concatenate([meas, [em]]))[0][:, 4:]).max() < 1e-8   # the same edge: the solves agree
    xo = R.oracle_optimize(X, ids2, np.concatenate([meas, [om]]))[0]   # the whole flow on the oracle: its alignment's mrad reaches 30 m out
    assert np.abs(xd[:, 4:] - xo[:, 4:]).max() < 3e-2
    assert np.linalg.norm(xo[-1, 4:] - truth[-1, 4:]) < before
    print(f"loop ({b}, {a}): alignment vs oracle {np.abs(np.array(K_dev[4:]) - np.array(K_orc[4:])).max():.2e} m, poses vs oracle "
          f"{np.abs(xd[:, 4:] - xo[:, 4:]).max():.2e} m, error of keyframe {b} {before:.3f} -> {np.linalg.norm(xd[-1, 4:] - truth[-1, 4:]):.3f} m")
    after = np.linalg.norm(xd[-1, 4:] - truth[-1, 4:])
    assert after < before, (before, after)


def test_search_gates_at_their_edges_on_the_device(ctx):
    """ll_loop_search's own gates at the edges, against the NumPy restatement: the keyframe difference exactly at the minimum, the nonzero
    ratios and the ROI difference exactly at the thresholds (and one float past), equal cell counts (a keyframe appended together with the newest),
    fewer cells than an earlier keyframe, a keyframe without line cells and an empty one (all-zero images: similarity 0)."""
    g, _ = _pair(ctx)
    r = np.random.default_rng(4)
    kfs = [Keyframe(ctx) for _ in range(6)]
    Keyframe.append(ctx, g, _scene(60, 6000), [kfs[0]])
    floor = np.c_[r.uniform(20, 26, 20000), r.uniform(0, 6, 20000), r.normal(0, 0.01, 20000), np.zeros(20000)].astype(np.float32)
    Keyframe.append(ctx, g, floor, [kfs[1]])                      # no line cells
    Keyframe.append(ctx, g, np.vstack([_scene(61, 6000, shift=(40, 0)), _scene(63, 6000, shift=(50, 0))]), [kfs[3]])   # more cells than the newest
    Keyframe.append(ctx, g, _scene(62, 6000, shift=(80, 0)), [kfs[4], kfs[5]])   # kfs[4] and the newest hold the same cells
    for kf in kfs:
        kf.analyze(g)                                             # kfs[2] stays empty
    infos = [kf.info() for kf in kfs]
    assert infos[1].line_cells == 0 and infos[2].cells == 0 and infos[4].cells == infos[5].cells < infos[3].cells
    cells = np.array([i.cells for i in infos], np.int64)
    roi = np.array([i.roi_range for i in infos], np.float32)
    rp = np.array([i.ratio_nonzero_plane for i in infos], np.float32)
    rl = np.array([i.ratio_nonzero_line for i in infos], np.float32)
    newest = 5
    loose = dict(K.DEFAULT_CFG, minimum_similarity_planar=-1.0, minimum_similarity_linear=-1.0, plane_with_line=-1.0, avail_ratio_plane=0.0,
                 avail_ratio_line=0.0, maximum_roi_difference=1e6, minimum_keyframe_differen=0)
    d0 = np.float32(abs(roi[0] - roi[newest]))
    cfgs = [loose,
            dict(loose, minimum_keyframe_differen=newest + 1 - 3), dict(loose, minimum_keyframe_differen=newest + 1 - 3 + 1),
            dict(loose, avail_ratio_plane=float(rp[0]), avail_ratio_line=float(rl[0])),
            dict(loose, avail_ratio_plane=float(np.nextafter(rp[0], np.float32(1))), avail_ratio_line=float(np.nextafter(rl[0], np.float32(1)))),
            dict(loose, maximum_roi_difference=float(d0)), dict(loose, maximum_roi_difference=float(np.nextafter(d0, np.float32(0)))),
            K.DEFAULT_CFG, dict(K.DEFAULT_CFG, minimum_keyframe_differen=1)]
    seen = set()
    for cfg in cfgs:
        sp, sl, cand = loop_search(ctx, kfs, newest, capi.default_loop_cfg(**cfg))
        assert cand == K.numpy_gates(cells, roi, rp, rl, np.c_[sp, sl], newest, cfg), cfg
        seen.add(tuple(cand))
        assert sp[2] == 0.0 and sl[2] == 0.0   # the empty keyframe's all-zero images
    # the cell-count line: only keyframes with at most the newest's cells and at least one pass; 4 (equal) does, 3 (more) and 2 (none) do not
    assert 4 in loose_cand(ctx, kfs, newest, loose) and 3 not in loose_cand(ctx, kfs, newest, loose) and 2 not in loose_cand(ctx, kfs, newest, loose)
    assert len(seen) >= 3


def loose_cand(ctx, kfs, newest, cfg):
    return loop_search(ctx, kfs, newest, capi.default_loop_cfg(**cfg))[2]


def test_keyframes_refuse_a_rebuilt_store(ctx):
    """A down-sample-and-replace assembly rewrites the store the keyframe's (slot, epoch) pairs point into: its analysis and appends are refused."""
    from loam_livox_b200.capi import LoamLivoxError
    g, _ = _pair(ctx)
    kf = Keyframe(ctx)
    Keyframe.append(ctx, g, _scene(70, 3000), [kf])
    kf.analyze(g)
    g.assemble(np.array([1.0, 0, 0, 0]), np.array([4.0, 3.0, 1.0]), 100.0, 180.0, 0.2, replace=True)
    with pytest.raises(LoamLivoxError):
        kf.analyze(g)
    with pytest.raises(LoamLivoxError):
        Keyframe.append(ctx, g, _scene(71, 3000), [kf])
    fresh = Keyframe(ctx)
    Keyframe.append(ctx, g, _scene(72, 3000), [fresh])
    assert fresh.analyze(g).cells > 0
