"""ll_register_batch on the GPU: several registrations against one map in one call, every item compared with ll_register of that item alone
(on a second context that never ran a batch) and with the oracle's registration of that item."""
import ctypes as C
import os

import numpy as np
import pytest

from loam_livox_b200 import synthetic as S

pytestmark = pytest.mark.gpu

INT_FIELDS = ("status", "registered", "icp_iterations", "num_residual_blocks", "corner_used", "surf_used", "total_lm_iterations", "total_evaluations")


@pytest.fixture(scope="module")
def ctxs():
    """(batch context, reference context): the reference only ever runs single registrations."""
    from loam_livox_b200.registration import Context
    b = Context(0, max_scan_points=400000, max_features=400000)
    r = Context(0, max_scan_points=400000, max_features=400000)
    yield b, r
    b.close(); r.close()


def _single(ctx, m, fc, fs, state):
    """ll_register of one item: (status code, RegResult)."""
    from loam_livox_b200 import capi
    from loam_livox_b200.capi import _pts
    c, fmt = _pts(fc); s, _ = _pts(fs)
    res = capi.RegResult()
    st = ctx._lib.ll_register(ctx.h, m.h, c.ctypes.data, c.shape[0], s.ctypes.data, s.shape[0], fmt, capi.LL_HOST, C.byref(state), C.byref(res))
    assert st in (capi.LL_OK, capi.LL_ERR_NO_BLOCKS), (st, ctx._lib.ll_last_error(ctx.h))
    return st, res


def _fields(r):
    return {n: (tuple(getattr(r, n)) if isinstance(getattr(r, n), C.Array) else getattr(r, n)) for n, _ in r._fields_ if not n.startswith("gpu_ms")}


def _state(pose, **kw):
    from loam_livox_b200 import capi
    return capi.default_reg_state(q_w_last=pose.q, t_w_last=pose.t, q_w_curr=pose.q, t_w_curr=pose.t, **kw)


def _assert_bit_identical(ctxs, m, fc, fs, state):
    from loam_livox_b200.registration import register_batch
    b, r = ctxs
    st1, r1 = _single(r, m, fc, fs, state)
    res, status = register_batch(b, m, [(fc, fs)], [state])
    assert status == [st1] and _fields(res[0]) == _fields(r1)
    return r1


# ---------------------------------------------------------------------------------------------- n = 1 is ll_register
def test_one_item_is_ll_register_golden(ctxs):
    from loam_livox_b200.registration import Map
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "golden_small.npz"))
    m = Map(ctxs[0], g["map_corner"], g["map_surf"])
    guess = S.Pose(g["guess_q"], g["guess_t"])
    r1 = _assert_bit_identical(ctxs, m, g["feat_corner"], g["feat_surf"], _state(guess))
    assert r1.registered == 1 and np.linalg.norm(np.array(r1.t_w_curr) - g["reg_t"]) < 1e-7


def test_one_item_is_ll_register_c2_size(ctxs):
    """A scan of the benchmark's C2 workload (100k-point scan, 5M-point map, the bench's pipeline leaves), its features from the library's front end."""
    import bench
    from loam_livox_b200.registration import Livox_laser, Map, voxel_grid_filter
    mc, ms, scans, guesses, _ = bench.make_inputs(0, "c2")
    m = Map(ctxs[0], mc, ms)
    lx = Livox_laser(ctxs[0])
    lx.extract_laser_features(scans[0], 100.0)
    c, s, _ = lx.get_features(0.0, 1.0)
    P = bench.PIPE
    c = voxel_grid_filter(ctxs[0], voxel_grid_filter(ctxs[0], c, P["extractor_leaf_corner"]), P["mapping_leaf_corner"])
    s = voxel_grid_filter(ctxs[0], voxel_grid_filter(ctxs[0], s, P["extractor_leaf_surf"]), P["mapping_leaf_surf"])
    assert c.shape[0] + s.shape[0] > 20000
    r1 = _assert_bit_identical(ctxs, m, c, s, _state(guesses[0]))
    assert r1.registered == 1 and r1.status == 1


@pytest.mark.parametrize("cap,seed", [(200, 7), (150, 3)])
def test_one_item_is_ll_register_capped(ctxs, cap, seed):
    from loam_livox_b200.registration import Map
    mc, ms = S.make_map(5000, 45000)
    pose = S.default_pose()
    fc, fs = S.make_features(1000, 9000, pose)
    m = Map(ctxs[0], mc, ms)
    guess = S.perturb_pose(pose, np.random.default_rng(seed))
    _assert_bit_identical(ctxs, m, fc, fs, _state(guess, maximum_allow_residual_block=cap, rng_seed=seed))


def test_one_item_is_ll_register_deblur(ctxs):
    from loam_livox_b200.registration import Map
    mc, ms = S.make_map(5000, 45000)
    m = Map(ctxs[0], mc, ms)
    last = S.default_pose()
    curr = S.Pose(S.quat_mul(last.q, S.quat_from_euler(0.01, -0.02, 0.06)), last.t + np.array((0.20, -0.05, 0.02)))
    fc, fs = S.make_distorted_features(last, curr, 1000, 9000, seed=0)
    r1 = _assert_bit_identical(ctxs, m, fc, fs, _state(last, if_motion_deblur=1))
    assert r1.registered == 1


# ---------------------------------------------------------------------------------------------- mixed batches
def _pool():
    """16 items against one map: different scans and initial poses, caps 200 / 150 / 1e6 with different seeds, one item under the :199 gate,
    one item stopped after 1 ICP iteration, items that never converge and run to their maximum, one item whose features all fail the match
    gates, and one scan under three initial guesses."""
    mc, ms = S.make_map(20000, 180000)
    base = S.default_pose()
    scans = []
    for k in range(5):
        pose = S.Pose(S.quat_mul(base.q, S.quat_from_euler(0.01 * k, -0.01 * k, 0.04 * k)), base.t + np.array([0.3 * k, -0.2 * k, 0.05 * k]))
        fc, fs = S.make_features(600 + 150 * k, 5400 + 900 * k, pose, seed=S.SEED + 31 * k)
        scans.append((fc, fs, pose))
    far = tuple(np.concatenate([a[:, :3] + 1000.0, a[:, 3:]], axis=1).astype(np.float32) for a in scans[1][:2])   # nothing of the map within the gates
    spec = [  # (scan, guess seed, extra state)
        (0, 0, {}), (0, 1, {}), (0, 2, {}),                                               # one scan, three guesses
        (1, 3, dict(maximum_allow_residual_block=200, rng_seed=3)),
        (2, 4, dict(maximum_allow_residual_block=150, rng_seed=4)),
        (1, 5, dict(current_frame_index=10)),                                             # :199 gate
        (2, 6, dict(icp_max_iterations=1)),
        ("far", 7, {}),                                                                   # LL_ERR_NO_BLOCKS alone
        (3, 8, dict(minimum_icp_R_diff=0.0, minimum_icp_T_diff=0.0, icp_max_iterations=6)),  # never converges: runs to its maximum
        (4, 9, dict(maximum_allow_residual_block=200, rng_seed=9)),
        (3, 10, dict(maximum_allow_residual_block=150, rng_seed=10)),
        (4, 11, dict(maximum_allow_residual_block=1000000, rng_seed=11)),
        (0, 12, dict(maximum_allow_residual_block=200, rng_seed=12, minimum_icp_R_diff=0.0, minimum_icp_T_diff=0.0)),   # runs to 15
        (1, 13, {}),
        (2, 14, dict(maximum_allow_residual_block=200, rng_seed=14)),
        (3, 15, {}),
    ]
    items = []
    for sc, seed, kw in spec:
        fc, fs, pose = (far[0], far[1], scans[1][2]) if sc == "far" else scans[sc]
        guess = S.perturb_pose(pose, np.random.default_rng(seed))
        items.append((fc, fs, guess, kw))
    return mc, ms, items


@pytest.fixture(scope="module")
def pool(ctxs):
    from loam_livox_b200.registration import Map
    mc, ms, items = _pool()
    m = Map(ctxs[0], mc, ms)
    singles = [_single(ctxs[1], m, fc, fs, _state(g, **kw)) for fc, fs, g, kw in items]
    return mc, ms, m, items, singles, {}


def _oracle_result(oracle, pool, k):
    mc, ms, _, items, _, cache = pool
    if k not in cache:
        if "trees" not in cache:
            cache["trees"] = (oracle.KdTree(mc), oracle.KdTree(ms))
        fc, fs, g, kw = items[k]
        p = oracle.default_params(q_w_last=g.q, t_w_last=g.t, q_w_curr=g.q, t_w_curr=g.t, **kw)
        cache[k] = oracle.register(mc, cache["trees"][0], ms, cache["trees"][1], fc, fs, p)
    return cache[k]


BATCHES = {2: [4, 6], 5: [0, 1, 2, 5, 7], 16: list(range(16))}


@pytest.mark.parametrize("n", [2, 5, 16])
def test_mixed_batch_matches_each_item_alone(ctxs, pool, oracle, n):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import register_batch
    _, _, m, items, singles, _ = pool
    ks = BATCHES[n]
    res, status = register_batch(ctxs[0], m, [items[k][:2] for k in ks], [_state(items[k][2], **items[k][3]) for k in ks])
    for j, k in enumerate(ks):
        st1, r1 = singles[k]
        r = res[j]
        assert status[j] == st1, (k, status[j], st1)
        assert tuple(getattr(r, f) for f in INT_FIELDS) == tuple(getattr(r1, f) for f in INT_FIELDS), (k, _fields(r), _fields(r1))
        # (component differences: quat_angle's acos resolves nothing below ~1.5e-8)
        assert np.abs(np.array(r.t_w_curr) - np.array(r1.t_w_curr)).max() <= 1e-9 and np.abs(np.array(r.q_w_curr) - np.array(r1.q_w_curr)).max() <= 1e-9, k
        if st1 != capi.LL_OK or r1.registered == 0:
            continue
        ost, ores = _oracle_result(oracle, pool, k)
        assert r.status == ost and r.icp_iterations == ores.icp_iterations, k
        assert np.linalg.norm(np.array(r.t_w_curr) - np.array(ores.t_w_curr)) < 1e-7 and S.quat_angle(np.array(r.q_w_curr), np.array(ores.q_w_curr)) < 1e-7, k
    if n >= 5:   # the mix really covers what it claims
        by = {k: (status[j], res[j]) for j, k in enumerate(ks)}
        assert by[7][0] == capi.LL_ERR_NO_BLOCKS and by[5][1].registered == 0
        if n == 16:
            assert by[6][1].icp_iterations == 1 and by[8][1].icp_iterations == 6 and by[12][1].icp_iterations == 15
            assert len({by[k][1].gpu_ms_total for k in ks if by[k][0] == capi.LL_OK and by[k][1].registered}) == 1   # the batch's timings


def test_batch_is_deterministic_and_leaves_single_calls_intact(ctxs, pool):
    from loam_livox_b200.registration import register_batch
    _, _, m, items, singles, _ = pool
    args = ([it[:2] for it in items], [_state(it[2], **it[3]) for it in items])
    a, sa = register_batch(ctxs[0], m, *args)
    b, sb = register_batch(ctxs[0], m, *args)
    assert sa == sb and [_fields(x) for x in a] == [_fields(x) for x in b]
    for k in (0, 3, 7):   # after a batch, ll_register on the same context is the fresh context's, bit for bit
        st, r = _single(ctxs[0], m, items[k][0], items[k][1], _state(items[k][2], **items[k][3]))
        assert st == singles[k][0] and _fields(r) == _fields(singles[k][1])


# ---------------------------------------------------------------------------------------------- edges
def _group_ctas(T, n, M):
    """batch_grid's group sizes (solve.cu): T CTAs at most, one each, the rest in proportion to the slots."""
    tot = sum(max(x, 1) for x in M)
    return [1 + (T - n) * max(x, 1) // tot for x in M]


def test_capacity_of_a_one_cta_group(ctxs):
    """The largest slot count that fits one CTA's shared memory (12 tiles of 256 slots: 3072) in a group of one CTA runs; one slot more is
    LL_ERR_CAPACITY before anything is enqueued."""
    import torch
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import LoamLivoxError, Map, register_batch
    T = min(torch.cuda.get_device_properties(0).multi_processor_count, 160)
    n, big = 16, 3072
    X = ((T - n - 1) * (big + 1)) // (n - 1) + 1 + 8   # the other 15 items: large enough that the 3073-slot item still gets one CTA
    for M0 in (big, big + 1):
        assert _group_ctas(T, n, [M0] + [X] * (n - 1))[0] == 1
    mc, ms = S.make_map(20000, 180000)
    m = Map(ctxs[0], mc, ms)
    pose = S.default_pose()
    others = [S.make_features(X // 10, X - X // 10, pose, seed=S.SEED + k) for k in range(2)]
    for M0, ok in ((big, True), (big + 1, False)):
        first = S.make_features(M0 // 10, M0 - M0 // 10, pose, seed=S.SEED + 5)
        items = [first] + [others[k % 2] for k in range(n - 1)]
        assert sum(a.shape[0] + b.shape[0] for a, b in items) <= 400000
        states = [_state(S.perturb_pose(pose, np.random.default_rng(k)), icp_max_iterations=2) for k in range(n)]
        l0 = ctxs[0].launches()
        if ok:
            res, status = register_batch(ctxs[0], m, items, states)
            assert status == [capi.LL_OK] * n and all(r.registered == 1 for r in res)
        else:
            with pytest.raises(LoamLivoxError, match=r"status -3: item 0:"):
                register_batch(ctxs[0], m, items, states)
            assert ctxs[0].launches() == l0


def test_total_features_at_max_features():
    from loam_livox_b200.registration import Context, LoamLivoxError, Map, register_batch
    ctx = Context(0, max_scan_points=20000, max_features=20000)
    mc, ms = S.make_map(5000, 45000)
    m = Map(ctx, mc, ms)
    pose = S.default_pose()
    fc, fs = S.make_features(1000, 9000, pose)
    st = _state(S.perturb_pose(pose, np.random.default_rng(0)))
    res, status = register_batch(ctx, m, [(fc, fs), (fc, fs)], [st, st])       # exactly max_features
    assert status == [0, 0] and res[0].registered == 1 and _fields(res[0]) == _fields(res[1])
    with pytest.raises(LoamLivoxError, match="status -3"):
        register_batch(ctx, m, [(fc, fs), (fc, np.concatenate([fs, fs[:1]]))], [st, st])
    ctx.close()


def test_whole_call_errors(ctxs):
    from loam_livox_b200 import capi
    from loam_livox_b200.registration import LoamLivoxError, Map, register_batch
    mc, ms = S.make_map(5000, 45000)
    m = Map(ctxs[0], mc, ms)
    pose = S.default_pose()
    fc, fs = S.make_features(200, 1800, pose)
    st = _state(pose)
    for n in (0, 17):
        with pytest.raises(LoamLivoxError, match="status -1"):
            register_batch(ctxs[0], m, [(fc, fs)] * n, [st] * n)
    with pytest.raises(LoamLivoxError, match="status -1: item 1: if_motion_deblur"):
        register_batch(ctxs[0], m, [(fc, fs)] * 2, [st, _state(pose, if_motion_deblur=1)])
    sharded = Map(ctxs[0], mc, ms, rank=0, world=2)
    with pytest.raises(LoamLivoxError, match="status -1"):
        register_batch(ctxs[0], sharded, [(fc, fs)], [st])
    res, status = register_batch(ctxs[0], m, [(fc, fs)], [st])   # the context is still usable
    assert status == [capi.LL_OK] and res[0].registered == 1
