"""Pose graph without a GPU: the NumPy restatement against complex-step derivatives and the oracle's Jets, the oracle's solver against
scipy.optimize.least_squares, its skyline factorization against numpy.linalg.solve, the host build of the device elimination against
numpy.linalg.solve in long double, and the C-ABI surface."""
import ctypes as C

import numpy as np
import pytest
import scipy.optimize

import pose_graph_reference as R


def _spd6(rng):
    A = rng.normal(size=(6, 6))
    return A @ A.T + 0.5 * np.eye(6)


def _jac_cases():
    rng = np.random.default_rng(1)
    for case in range(12):
        xa = np.concatenate([R.random_quat(rng, 2.0), rng.normal(size=3)])
        xb = np.concatenate([R.random_quat(rng, 2.0), rng.normal(size=3)])
        meas = np.concatenate([R.random_quat(rng, 2.0), rng.normal(size=3)])
        W = None
        if case % 4 == 1:   # 180 degree relative rotation
            xb[:4] = R.qmul(xa[:4], np.array([0.0, 0.0, 0.0, 1.0]))
        if case % 4 == 2:   # -q and far poses
            xb[:4] = -xb[:4]
            xa[4:7] += 1e4
            xb[4:7] -= 1e4
        if case % 4 == 3:
            W = _spd6(rng)
        yield xa, xb, meas, W


@pytest.mark.parametrize("k", range(12))
def test_jacobian_analytic_vs_complex_step_and_oracle(k):
    xa, xb, meas, W = list(_jac_cases())[k]
    Ja_c, Jb_c = R.jacobian_complex_step(xa, xb, meas, W)
    Ja_a, Jb_a = R.jacobian_analytic(xa, xb, meas, W)
    r_o, Ja_o, Jb_o = R.oracle_residual(xa, xb, meas, W)
    scale = max(1.0, np.abs(Ja_c).max(), np.abs(Jb_c).max())
    for J1, J2 in ((Ja_a, Ja_c), (Jb_a, Jb_c), (Ja_o, Ja_c), (Jb_o, Jb_c)):
        assert np.abs(np.asarray(J1, np.float64) - J2).max() <= 1e-12 * scale
    assert np.allclose(r_o, R.residual(xa, xb, meas, W), rtol=0, atol=1e-12 * max(1.0, np.abs(xa[4:]).max()))
    if W is not None:   # L, not L^T and not the symmetric square root
        assert not np.allclose(R.sqrt_information(W), R.sqrt_information(W).T)
        e = R.error6(xa, xb, meas)
        assert np.allclose(r_o, R.sqrt_information(W) @ e) and not np.allclose(r_o, R.sqrt_information(W).T @ e)


def _flat_residuals(z, X0, ids, meas, free):
    X = X0.copy()
    for j, n in enumerate(free):
        X[n] = R.plus(X0[n], z[6 * j:6 * j + 6])
    return np.concatenate([R.residual(X[a], X[b], meas[e]) for e, (a, b) in enumerate(ids)])


@pytest.mark.parametrize("n,loops", [(5, [(4, 0)]), (20, [(19, 2), (10, 0)]), (50, [(49, 0), (30, 5)])])
def test_oracle_optimum_matches_least_squares(n, loops):
    rng = np.random.default_rng(n)
    truth = R.trajectory(n, rng)
    X, ids, meas = R.chain_graph(truth, rng, loops)
    xo, c0, c1, it, ev, term = R.oracle_optimize(X, ids, meas)
    assert term in (1, 2, 3) and c1 < c0
    free = list(range(1, n))
    sol = scipy.optimize.least_squares(_flat_residuals, np.zeros(6 * len(free)), args=(xo, ids, meas, free), xtol=1e-15, ftol=1e-15, gtol=1e-15)
    # ceres stops on its function tolerance (|cost change| <= 1e-6 cost), not at the exact optimum: the optimum found from the oracle's poses
    # is within that relative cost of the oracle's (the poses themselves may differ along directions the cost hardly sees)
    cost_o = 0.5 * np.sum(_flat_residuals(np.zeros(6 * len(free)), xo, ids, meas, free) ** 2)
    assert abs(cost_o - c1) <= 1e-12 * c1
    assert sol.cost <= cost_o and cost_o - sol.cost <= 1e-6 * cost_o


@pytest.mark.parametrize("n,loops", [(10, [(9, 0)]), (30, [(29, 3), (20, 0)])])
def test_oracle_poses_at_the_least_squares_optimum(n, loops):
    """With its function and parameter tolerances tightened to 1e-15 (everything else as ceres has it) the oracle runs to the optimum itself:
    its poses are those of scipy.optimize.least_squares' optimum within 1e-8 m and 1e-8 rad."""
    rng = np.random.default_rng(100 + n)
    truth = R.trajectory(n, rng)
    X, ids, meas = R.chain_graph(truth, rng, loops)
    xo, c0, c1, it, ev, term = R.oracle_optimize(X, ids, meas, ftol=1e-15, ptol=1e-15)
    assert term in (1, 2, 3) and it < 200
    free = list(range(1, n))
    # least_squares (LM) started at the oracle's poses reaches its own optimum within 1e-8 m / rad of them
    sol = scipy.optimize.least_squares(_flat_residuals, np.zeros(6 * len(free)), args=(xo, ids, meas, free), xtol=1e-15, ftol=1e-15, gtol=1e-15,
                                       method="lm")
    assert sol.cost <= 0.5 * np.sum(_flat_residuals(np.zeros(6 * len(free)), xo, ids, meas, free) ** 2) * (1 + 1e-12)
    assert np.abs(sol.x).max() <= 1e-8


def test_non_finite_initial_cost_reports_it():
    X = np.array([[1.0, 0, 0, 0, 0, 0, 0], [1.0, 0, 0, 0, 1e200, 0, 0]])
    ids = np.array([[0, 1]], np.int32)
    meas = np.array([[1.0, 0, 0, 0, -1e200, 0, 0]])
    xo, c0, c1, it, ev, term = R.oracle_optimize(X, ids, meas)
    assert term == 4 and it == 0 and np.isinf(c0) and np.isinf(c1) and np.array_equal(xo, X)


def test_consistent_chain_stops_on_the_gradient_test():
    rng = np.random.default_rng(3)
    truth = R.trajectory(30, rng)
    ids = np.array([(i, i + 1) for i in range(29)], np.int32)
    meas = np.array([R.relative(truth[i], truth[i + 1]) for i in range(29)])
    xo, c0, c1, it, ev, term = R.oracle_optimize(truth, ids, meas)
    assert term == 1 and it == 0 and ev == 1 and c0 < 1e-20
    assert np.array_equal(xo, truth)


def test_skyline_solve_matches_numpy():
    rng = np.random.default_rng(4)
    for n in (1, 6, 30, 61):
        B = rng.normal(size=(n, n)) * (rng.random((n, n)) < 0.2)
        A = B @ B.T + n * np.eye(n)
        b = rng.normal(size=n)
        assert np.allclose(R.skyline_solve(A, b), np.linalg.solve(A, b), rtol=1e-12, atol=1e-12)


def _graph_system(N, ids, rng, lam=0.1):
    """A = sum over edges of J^T J for a random J per edge, + lam I on every free node: the shape of the LM normal equations."""
    free = sorted({int(v) for e in ids for v in e} - {0})
    node = np.zeros((N, 6, 6))
    edge = np.zeros((len(ids), 6, 6))
    for e, (a, b) in enumerate(ids):
        Ja, Jb = rng.normal(size=(6, 6)), rng.normal(size=(6, 6))
        node[a] += Ja.T @ Ja
        node[b] += Jb.T @ Jb
        edge[e] = Ja.T @ Jb
    for f in free:
        node[f] += lam * np.eye(6)
    rhs = rng.normal(size=(N, 6))
    idx = {f: k for k, f in enumerate(free)}
    A = np.zeros((6 * len(free), 6 * len(free)), np.longdouble)
    for f in free:
        A[6 * idx[f]:6 * idx[f] + 6, 6 * idx[f]:6 * idx[f] + 6] = node[f]
    for e, (a, b) in enumerate(ids):
        if a in idx and b in idx:
            A[6 * idx[a]:6 * idx[a] + 6, 6 * idx[b]:6 * idx[b] + 6] += edge[e]
            A[6 * idx[b]:6 * idx[b] + 6, 6 * idx[a]:6 * idx[a] + 6] += edge[e].T
    bv = np.concatenate([rhs[f] for f in free]).astype(np.longdouble)
    return node, edge, rhs, A, bv, free


def _shapes():
    yield "one segment per length", 40, [(i, i + 1) for i in range(39)]
    for L in (1, 2, 3, 7, 8, 9, 15, 16, 17, 31, 33):   # 2^k +- 1
        yield f"length {L} between two border nodes", L + 3, [(i, i + 1) for i in range(L + 2)] + [(1, L + 2)]
    yield "no border, reversed and duplicate edges", 12, [(i + 1, i) for i in range(11)] + [(3, 4), (4, 3)]
    yield "adjacent border nodes", 12, [(i, i + 1) for i in range(11)] + [(2, 5), (3, 9), (4, 11)]
    yield "nodes without edges", 20, [(i, i + 1) for i in range(5)] + [(9, 10), (10, 11), (15, 16), (16, 19)]
    yield "edges to node 0", 10, [(i, i + 1) for i in range(9)] + [(0, 5), (7, 0)]
    yield "border of 64", 200, [(i, i + 1) for i in range(199)] + [(3 * k + 2, 199 - 3 * k) for k in range(32)]


@pytest.mark.parametrize("name,N,edges", list(_shapes()), ids=[s[0] for s in _shapes()])
def test_host_elimination_backward_error(name, N, edges):
    rng = np.random.default_rng(N + len(edges))
    ids = np.array(edges, np.int32)
    node, edge, rhs, A, bv, free = _graph_system(N, ids, rng)
    x, nb, stats = R.host_solve(N, ids, node, edge, rhs)
    assert nb >= 0 and stats[0] == len(free)
    if name == "border of 64":
        assert nb == 64
    xv = np.concatenate([x[f] for f in free]).astype(np.longdouble)
    res = A @ xv - bv
    err = np.sqrt(np.sum(res * res)) / (np.linalg.norm(np.asarray(A, np.float64), 2) * np.sqrt(np.sum(xv * xv)))
    assert err <= 1e-14, err
    assert np.allclose(np.asarray(xv, np.float64), np.linalg.solve(np.asarray(A, np.float64), np.asarray(bv, np.float64)), rtol=1e-8, atol=1e-10)
    assert all(not x[n].any() for n in range(N) if n not in free)


def test_loop_edge_restatement_matches_oracle():
    rng = np.random.default_rng(5)
    for _ in range(10):
        qa, qb, qi = (R.random_quat(rng, 2.0) for _ in range(3))
        pa = np.concatenate([qa, rng.normal(size=3) * 10])
        pb = np.concatenate([qb, rng.normal(size=3) * 10])
        ti = rng.normal(size=3)
        q, t = R.loop_edge(qi * 1.001, ti, pa, pb)   # a non-unit ICP quaternion: inverse() divides by the squared norm
        (b, e), meas = R.oracle_loop_edge(qi * 1.001, ti, pa, 7, pb, 9)
        assert (b, e) == (9, 7)
        assert np.allclose(meas[:4], q, rtol=0, atol=1e-14) and np.allclose(meas[4:], t, rtol=0, atol=1e-12)


def test_cabi_surface():
    from loam_livox_b200 import capi
    L = capi.lib()
    for n in ("ll_pose_graph_create", "ll_pose_graph_release", "ll_pose_graph_optimize", "ll_pose_graph_step", "ll_pose_graph_loop_edge"):
        assert n in capi.EXPORTS and hasattr(L, n)
    assert C.sizeof(capi.Pose) == 56 and C.sizeof(capi.PgEdge) == 8 + 56 + 288 and C.sizeof(capi.PgSummary) == 16 + 8 * 4 + 4 * 8
    h = C.c_void_p()
    assert L.ll_pose_graph_create(None, 10, 10, C.byref(h)) == capi.LL_ERR_INVALID
    assert L.ll_pose_graph_optimize(None, None, 0, None, 0, 0, None) == capi.LL_ERR_INVALID
    L.ll_pose_graph_release(None)
    # the library's loop edge is the restatement's
    rng = np.random.default_rng(6)
    from loam_livox_b200.registration import pg_loop_edge
    pa = np.concatenate([R.random_quat(rng), rng.normal(size=3)])
    pb = np.concatenate([R.random_quat(rng), rng.normal(size=3)])
    qi, ti = R.random_quat(rng), rng.normal(size=3)
    e = pg_loop_edge(qi, ti, pa, 2, pb, 5)
    (b, a), meas = R.oracle_loop_edge(qi, ti, pa, 2, pb, 5)
    assert (e.id_begin, e.id_end) == (b, a) == (5, 2)
    assert np.array_equal(np.array(e.q_wxyz), meas[:4]) and np.array_equal(np.array(e.t), meas[4:])
    assert np.array_equal(np.array(e.information).reshape(6, 6), np.eye(6))
