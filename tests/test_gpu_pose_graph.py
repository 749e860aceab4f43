"""The device pose-graph solve (ll_pose_graph_optimize / ll_pose_graph_step) against the oracle (oracle/orc_pose_graph.hpp) and against a
long-double product, its refusals and limits, its determinism, the reference's loop-closure flow through ll_scene_align, and the re-posed
keyframe clouds (ll_keyframes_repose) bit for bit against the oracle."""
import ctypes as C

import numpy as np
import pytest

import pose_graph_reference as R
from loam_livox_b200 import capi
from loam_livox_b200 import synthetic as S
from loam_livox_b200.registration import Context, PoseGraph, Scene_alignment, keyframes_repose, pg_edges, pg_loop_edge

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = Context(0, max_scan_points=1000, max_features=1000)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pg(ctx):
    g = PoseGraph(ctx, 5000, 6000)
    yield g
    g.close()


def _edges(ids, meas, W=None):
    return pg_edges(ids[:, 0], ids[:, 1], meas[:, :4], meas[:, 4:7], W)


def _loops(n, k, rng):
    return [(int(b), int(a)) for a, b in zip(rng.integers(0, n // 3, k), rng.integers(2 * n // 3, n, k))]


def _case(n, k, seed, reverse=False, dup=False, W=None):
    rng = np.random.default_rng(seed)
    truth = R.trajectory(n, rng)
    X, ids, meas = R.chain_graph(truth, rng, _loops(n, k, rng) if k else ())
    if reverse:   # every other odometry edge runs backwards with the inverse measurement
        for e in range(0, n - 1, 2):
            a, b = ids[e]
            ids[e] = (b, a)
            meas[e] = R.relative(truth[b], truth[a])
    if dup:
        ids = np.concatenate([ids, ids[:3]])
        meas = np.concatenate([meas, meas[:3]])
    return X, ids, meas


def _parity(pg, X, ids, meas, W=None, max_iterations=200):
    Wm = None if W is None else np.broadcast_to(W, (ids.shape[0], 6, 6))
    xd, s = pg.optimize(X, _edges(ids, meas, Wm), max_iterations)
    xo, c0, c1, it, ev, term = R.oracle_optimize(X, ids, meas, Wm, max_iterations)
    assert (s.termination, s.iterations, s.evaluations) == (term, it, ev)
    assert abs(s.initial_cost - c0) <= 1e-10 * c0 and abs(s.final_cost - c1) <= 1e-10 * max(c1, 1e-300)
    assert np.abs(xd[:, 4:] - xo[:, 4:]).max() <= 1e-8
    ang = [R.qmul(R.conj(xo[i, :4]), xd[i, :4]) for i in range(X.shape[0])]
    assert max(2 * np.linalg.norm(a[1:]) for a in ang) <= 1e-8
    return xd, s


@pytest.mark.parametrize("n,k", [(2, 0), (3, 0), (3, 1), (10, 1), (300, 1), (300, 32), (5000, 1), (5000, 32), (1000, 32)])
def test_parity_with_oracle(pg, n, k):
    X, ids, meas = _case(n, k, seed=n + k)
    xd, s = _parity(pg, X, ids, meas)
    assert s.free_nodes == n - 1 and s.border_nodes <= 2 * k


def test_parity_variants(pg):
    rng = np.random.default_rng(7)
    W = rng.normal(size=(6, 6))
    W = W @ W.T + np.eye(6)
    _parity(pg, *_case(40, 2, 11, reverse=True))
    _parity(pg, *_case(40, 2, 12, dup=True))
    _parity(pg, *_case(40, 2, 13), W=W)
    for it in (1, 2):
        _parity(pg, *_case(60, 3, 14), max_iterations=it)
    # a loop to node 0 and poses no edge touches
    X, ids, meas = _case(30, 0, 15)
    keep = [e for e in range(ids.shape[0]) if not (10 <= ids[e].min() < 14)]
    ids, meas = np.concatenate([ids[keep], [[29, 0]]]), np.concatenate([meas[keep], [R.relative(X[29], X[0])]])
    xd, s = _parity(pg, X, ids, meas)
    assert np.array_equal(xd[11:14], X[11:14]) and np.array_equal(xd[0], X[0])


def _with_loops(n, loops, seed):
    rng = np.random.default_rng(seed)
    truth = R.trajectory(n, rng)
    return R.chain_graph(truth, rng, loops)


def test_border_limits_and_many_loop_edges(pg, ctx):
    """64 loop edges over 32 border poses; a border of exactly LL_PG_MAX_BORDER = 64 solved; 65 refused without a launch."""
    S32 = [10 * (i + 1) for i in range(32)]
    loops = [(S32[i % 32], S32[(7 * i + 5) % 32]) for i in range(64)]
    assert all(a != b for a, b in loops)
    X, ids, meas = _with_loops(400, loops, 60)
    xd, s = _parity(pg, X, ids, meas)
    assert s.border_nodes == 32
    loops64 = [(2 * i + 1, 399 - 2 * i) for i in range(32)]
    X, ids, meas = _with_loops(400, loops64, 61)
    xd, s = _parity(pg, X, ids, meas)
    assert s.border_nodes == 64 == capi.LL_PG_MAX_BORDER
    X, ids, meas = _with_loops(400, loops64 + [(1, 300)], 62)
    x = np.ascontiguousarray(X).copy()
    E = _edges(ids, meas)
    n0 = ctx.launches()
    st = capi.lib().ll_pose_graph_optimize(pg.h, x.ctypes.data, 400, C.cast(E, C.c_void_p), len(E), 0, C.byref(capi.PgSummary()))
    assert st == capi.LL_ERR_CAPACITY and "65 border nodes" in capi.lib().ll_last_error(ctx.h).decode()
    assert ctx.launches() == n0 and np.array_equal(x, X)


def test_step_backward_error(pg):
    for n, k in ((3, 1), (300, 32), (400, 16)):
        X, ids, meas = _case(n, k, 20 + n)
        for radius in (1e4, 1.0):
            cost, g, s, st, valid = pg.step(X, _edges(ids, meas), radius)
            assert valid
            L = np.longdouble
            A = np.zeros((6 * n, 6 * n), L)
            for e, (a, b) in enumerate(ids):
                Ja, Jb = R.jacobian_analytic(X[a], X[b], meas[e])
                for (u, Ju) in ((a, Ja), (b, Jb)):
                    for (v, Jv) in ((a, Ja), (b, Jb)):
                        if u and v:
                            A[6 * u:6 * u + 6, 6 * v:6 * v + 6] += Ju.T @ Jv
            A = A[6:, 6:]
            sv = s[1:].reshape(-1).astype(L)
            As = sv[:, None] * A * sv[None, :]
            D = np.clip(np.diag(As).astype(np.float64), 1e-6, 1e32)
            As[np.diag_indices_from(As)] += D / radius
            rhs = -(sv * g[1:].reshape(-1).astype(L))
            x = st[1:].reshape(-1).astype(L)
            res = As @ x - rhs
            err = np.sqrt(np.sum(res * res)) / (np.linalg.norm(np.asarray(As, np.float64), 2) * np.sqrt(np.sum(x * x)))
            assert err <= 1e-14, (n, k, radius, err)


def test_capacity_refusals_and_empty(pg, ctx):
    L = capi.lib()
    X, ids, meas = _case(400, 0, 30)
    loops = [(2 * i + 1, 399 - 2 * i) for i in range(33)]   # 66 border nodes
    ids2 = np.concatenate([ids, loops]).astype(np.int32)
    meas2 = np.concatenate([meas, [R.relative(X[a], X[b]) for a, b in loops]])
    x = np.ascontiguousarray(X).copy()
    E = _edges(ids2, meas2)
    s = capi.PgSummary()
    assert L.ll_pose_graph_optimize(pg.h, x.ctypes.data, 400, C.cast(E, C.c_void_p), len(E), 0, C.byref(s)) == capi.LL_ERR_CAPACITY
    assert np.array_equal(x, X)
    X, ids, meas = _case(20, 1, 31)
    n0 = ctx.launches()
    bad = []
    for mut in range(6):
        E = _edges(ids, meas)
        if mut == 0: E[3].id_end = 20
        if mut == 1: E[3].id_begin = -1
        if mut == 2: E[3].id_end = E[3].id_begin
        if mut == 3: E[3].t[1] = float("nan")
        if mut == 4: E[3].information[1] = 0.5   # not symmetric
        if mut == 5: E[3].information[0] = -1.0  # not positive definite
        x = np.ascontiguousarray(X).copy()
        bad.append(L.ll_pose_graph_optimize(pg.h, x.ctypes.data, 20, C.cast(E, C.c_void_p), len(E), 0, C.byref(s)))
        assert np.array_equal(x, X)
    assert bad == [capi.LL_ERR_INVALID] * 6 and ctx.launches() == n0   # nothing enqueued
    x = np.ascontiguousarray(X).copy()
    x[5, 4] = float("inf")
    E = _edges(ids, meas)
    assert L.ll_pose_graph_optimize(pg.h, x.ctypes.data, 20, C.cast(E, C.c_void_p), len(E), 0, C.byref(s)) == capi.LL_ERR_INVALID
    xd, s = pg.optimize(X, (capi.PgEdge * 0)())
    assert np.array_equal(xd, X) and s.iterations == 0 and s.evaluations == 0


def test_determinism(pg, ctx):
    X, ids, meas = _case(3000, 16, 40)
    a, _ = pg.optimize(X, _edges(ids, meas))
    b, _ = pg.optimize(X, _edges(ids, meas))
    c2 = Context(0, max_scan_points=1000, max_features=1000)
    g2 = PoseGraph(c2, 100, 100)
    c, _ = g2.optimize(X, _edges(ids, meas))
    g2.close()
    c2.close()
    assert np.array_equal(a, b) and np.array_equal(a, c)


def _comp(u, v):
    return np.concatenate([R.qmul(u[:4], v[:4]), u[4:] + R.qrot(u[:4], v[4:])])


def _inv(u):
    return np.concatenate([R.conj(u[:4]), -R.qrot(R.conj(u[:4]), u[4:])])


def _move(cloud, T):
    c = cloud.copy()
    Rm = S.quat_to_mat(T[:4])
    c[:, :3] = (c[:, :3].astype(np.float64) @ Rm.T + T[4:]).astype(np.float32)
    return c


def test_loop_closure_flow(pg, ctx):
    """The reference's flow (laser_mapping.hpp:1034-1089): two keyframe clouds of the synthetic room as the drifted map holds them (keyframe k's
    points at X_k T_k^-1 of the room, T the truth), aligned by ll_scene_align with the newer keyframe first (find_tranfrom_of_two_mappings(
    last_keyframe, keyframe_vec[his])), the loop edge built by ll_pose_graph_loop_edge, the drifted chain optimized.  The same flow on the
    oracle (its scene alignment, loop edge and solver) gives the same edge and poses; the loop keyframe's error against the truth falls."""
    from oracle import oracle as O
    rng = np.random.default_rng(70)
    n = 40
    truth = R.trajectory(n, rng, yaw=2 * np.pi / n)
    X, ids, meas = R.chain_graph(truth, rng, (), dt=0.01, da=0.003)
    a, b = 0, n - 1
    room_a = S.make_map(4000, 40000, seed=S.SEED + 80)
    room_b = S.make_map(4000, 40000, seed=S.SEED + 81)
    Da, Db = _comp(X[a], _inv(truth[a])), _comp(X[b], _inv(truth[b]))
    al, ap = (_move(c, Da) for c in room_a)
    bl, bp = (_move(c, Db) for c in room_b)
    before = np.linalg.norm(X[b, 4:] - truth[b, 4:])
    assert 0.05 < before < 0.5   # a drift the coarse-to-fine alignment starts from
    big = Context(0, max_scan_points=100000, max_features=100000)   # room for the target keyframe's features
    sa = Scene_alignment(big)
    r = sa.find_tranfrom_of_two_mappings(bl, bp, al, ap)
    big.close()
    ores, oruns = O.scene_align(bl, bp, al, ap, threads=8)
    assert r.registered == 1 and sa.scales_run == oruns == 3
    K = np.concatenate([np.array(r.q_w_curr), np.array(r.t_w_curr)])
    Ktrue = _comp(Db, _inv(Da))   # X_b T_b^-1 T_a X_a^-1: maps keyframe a's cloud onto keyframe b's
    assert np.linalg.norm(K[4:] - Ktrue[4:]) < 0.05 and S.quat_angle(K[:4], Ktrue[:4]) < 0.01
    e = pg_loop_edge(K[:4], K[4:], X[a], a, X[b], b)
    (ob, oa), om = R.oracle_loop_edge(np.array(ores.q_w_curr), np.array(ores.t_w_curr), X[a], a, X[b], b)
    em = np.concatenate([np.array(e.q_wxyz), np.array(e.t)])
    assert (e.id_begin, e.id_end) == (ob, oa) == (b, a)
    assert np.abs(em - om).max() < 1e-5   # the two alignments agree to 1e-6 (test_scene_alignment_parity)
    assert np.linalg.norm(em[4:] - R.relative(truth[b], truth[a])[4:]) < 0.05
    ids2 = np.concatenate([ids, [[b, a]]]).astype(np.int32)
    xd, s = _parity(pg, X, ids2, np.concatenate([meas, [em]]))   # the device solve equals the oracle's on the device's edge
    xo = R.oracle_optimize(X, ids2, np.concatenate([meas, [om]]))[0]   # the whole flow on the oracle
    assert np.abs(xd[:, 4:] - xo[:, 4:]).max() < 1e-4
    after = np.linalg.norm(xd[b, 4:] - truth[b, 4:])
    assert after * 3 <= before, (before, after)


def _clouds(rng, sizes, nan_at=()):
    out = []
    for k, m in enumerate(sizes):
        c = np.concatenate([rng.normal(size=(m, 3)) * 3 + rng.normal(size=3) * 20, rng.random((m, 1)) * 100], axis=1).astype(np.float32)
        if k in nan_at and m:
            c[::7, 0] = np.nan
        out.append(c)
    return out


@pytest.mark.parametrize("sizes,nan_at", [((3000, 0, 2500, 40), (2,)), ((200,) * 256, (0, 255))], ids=["several keyframes, an empty one, NaN", "256 keyframes"])
def test_keyframes_repose_bit_exact(ctx, sizes, nan_at):
    rng = np.random.default_rng(len(sizes))
    clouds = _clouds(rng, sizes, nan_at)
    n = len(sizes)
    ori = np.array([np.concatenate([R.random_quat(rng, 2.0), rng.normal(size=3) * 30]) for _ in range(n)])
    opt = np.array([np.concatenate([R.qmul(ori[k, :4], R.random_quat(rng, 0.05)), ori[k, 4:] + rng.normal(size=3)]) for k in range(n)])
    got = keyframes_repose(ctx, clouds, ori, opt, 0.4)
    ref, cnt = R.oracle_repose(np.concatenate(clouds), np.cumsum(sizes), ori, opt, 0.4)
    assert [g.shape[0] for g in got] == list(cnt)
    assert np.array_equal(np.concatenate(got), ref)
    assert got[0].shape[0] > 0 and np.all(np.isfinite(np.concatenate(got)))
    if sizes[1] == 0:
        assert got[1].shape[0] == 0


def test_keyframes_repose_refuses_257(ctx):
    rng = np.random.default_rng(3)
    clouds = _clouds(rng, (10,) * 257)
    poses = np.tile([1.0, 0, 0, 0, 0, 0, 0], (257, 1))
    n0 = ctx.launches()
    with pytest.raises(capi.LoamLivoxError):
        keyframes_repose(ctx, clouds, poses, poses, 0.4)
    assert ctx.launches() == n0
