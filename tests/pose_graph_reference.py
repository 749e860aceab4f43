"""NumPy restatement of the pose graph (ceres_pose_graph_3d.hpp:198-352): the residual, the tangent-space Jacobian, ceres'
EigenQuaternionParameterization::Plus and the loop edge of Scene_alignment::add_constrain_of_loop.  Poses are rows (qw, qx, qy, qz, tx, ty, tz).

Also builds the two host libraries the tests use: the oracle (oracle/orc_pose_graph.hpp) and the host build of the device elimination
(loam_livox_b200/csrc/pg_plan.h, pg_block.cuh)."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def qmul(a, b):
    return np.array([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
                     a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                     a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3],
                     a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1]])


def qrot(q, v):
    """Eigen's _transformVector (valid as a rotation for unit q)."""
    u = np.array(q[1:4])
    c = 2 * np.cross(u, v)
    return v + q[0] * c + np.cross(u, c)


def conj(q):
    return np.array([q[0], -q[1], -q[2], -q[3]])


def error6(xa, xb, meas):
    """PoseGraph3dErrorTerm before the sqrt-information product."""
    qa, pa, qb, pb = xa[:4], xa[4:7], xb[:4], xb[4:7]
    ep = qrot(conj(qa), pb - pa) - meas[4:7]
    d = qmul(meas[:4], conj(qmul(conj(qa), qb)))
    return np.concatenate([ep, 2 * d[1:4]])


def sqrt_information(W):
    return np.linalg.cholesky(np.asarray(W, np.float64))   # lower factor L, W = L L^T


def residual(xa, xb, meas, W=None):
    e = error6(xa, xb, meas)
    return e if W is None else sqrt_information(W) @ e


def plus(x, d):
    """EigenQuaternionParameterization::Plus on q, Euclidean on t; d = (position 3, rotation 3).  Also valid for complex d (complex step)."""
    d = np.asarray(d)
    nd = np.sqrt(d[3] ** 2 + d[4] ** 2 + d[5] ** 2)
    if np.all(d[3:6] == 0):
        q = np.array(x[:4], dtype=np.result_type(x, d))
    else:
        s = np.sin(nd) / nd
        q = qmul(np.array([np.cos(nd), s * d[3], s * d[4], s * d[5]]), x[:4])
    return np.concatenate([q, x[4:7] + d[:3]])


def jacobian_complex_step(xa, xb, meas, W=None, h=1e-30):
    """Tangent-space Jacobian blocks (6 x 6 each) by complex-step differentiation through Plus."""
    Ja, Jb = np.zeros((6, 6)), np.zeros((6, 6))
    for k in range(6):
        d = np.zeros(6, complex)
        d[k] = 1j * h
        Ja[:, k] = residual(plus(xa.astype(complex), d), xb.astype(complex), meas, W).imag / h
        Jb[:, k] = residual(xa.astype(complex), plus(xb.astype(complex), d), meas, W).imag / h
    return Ja, Jb


def jacobian_analytic(xa, xb, meas, W=None):
    """The same blocks analytically in long double: a unit tangent e_k moves q by (0, e_k) q (Plus at delta = 0)."""
    L = np.longdouble
    xa, xb, meas = xa.astype(L), xb.astype(L), meas.astype(L)
    qa, pa, qb, pb, qm = xa[:4], xa[4:7], xb[:4], xb[4:7], meas[:4]
    qac, dp = conj(qa), pb - pa
    Ja, Jb = np.zeros((6, 6), L), np.zeros((6, 6), L)
    for k in range(3):
        e = np.zeros(3, L)
        e[k] = 1
        pk = np.concatenate([[L(0)], e])
        col = qrot(qac, e)
        Jb[:3, k], Ja[:3, k] = col, -col
        Jb[3:, 3 + k] = 2 * qmul(qm, conj(qmul(qac, qmul(pk, qb))))[1:4]
        dqac = conj(qmul(pk, qa))
        u, du = qac[1:4], dqac[1:4]
        c, dc = 2 * np.cross(u, dp), 2 * np.cross(du, dp)
        Ja[:3, 3 + k] = dqac[0] * c + qac[0] * dc + np.cross(du, c) + np.cross(u, dc)
        Ja[3:, 3 + k] = 2 * qmul(qm, conj(qmul(dqac, qb)))[1:4]
    if W is not None:
        S = sqrt_information(W).astype(L)
        Ja, Jb = S @ Ja, S @ Jb
    return Ja, Jb


def qinv(q):
    """Eigen's Quaternion::inverse(): the conjugate over the squared norm."""
    n2 = (q[1] * q[1] + q[3] * q[3]) + (q[2] * q[2] + q[0] * q[0])
    return conj(q) / n2


def loop_edge(icp_q, icp_t, pose_a, pose_b):
    """(q, t) of add_constrain_of_loop after laser_mapping.hpp:1065-1066's inversion; the edge runs from b (begin) to a (end)."""
    iq = qinv(np.asarray(icp_q, np.float64))
    it = qrot(iq, -np.asarray(icp_t, np.float64))
    qbi, iqi = qinv(pose_b[:4]), qinv(iq)
    q = qmul(qmul(qbi, iqi), pose_a[:4])
    t = qrot(qbi, qrot(iqi, pose_a[4:7] - it) - pose_b[4:7])
    return q, t


def random_quat(rng, scale=1.0):
    v = rng.normal(size=3) * scale
    a = np.linalg.norm(v)
    return np.concatenate([[np.cos(a / 2)], np.sin(a / 2) * v / a]) if a > 0 else np.array([1.0, 0, 0, 0])


def relative(xa, xb):
    """The measurement that makes the edge a -> b consistent: (conj(q_a) q_b, conj(q_a) (p_b - p_a))."""
    return np.concatenate([qmul(conj(xa[:4]), xb[:4]), qrot(conj(xa[:4]), xb[4:7] - xa[4:7])])


def trajectory(n, rng, step=1.0, yaw=0.05):
    """Keyframe poses along a planar loop with small tilts: rows (q, t)."""
    X = np.zeros((n, 7))
    X[0, 0] = 1.0
    for i in range(1, n):
        dq = qmul(random_quat(rng, 0.01), np.array([np.cos(yaw / 2), 0, 0, np.sin(yaw / 2)]))
        X[i, :4] = qmul(X[i - 1, :4], dq)
        X[i, :4] /= np.linalg.norm(X[i, :4])
        X[i, 4:7] = X[i - 1, 4:7] + qrot(X[i - 1, :4], np.array([step, 0, 0.01 * rng.normal()]))
    return X


def noisy(meas, rng, dt=0.02, da=0.005):
    q = qmul(meas[:4], random_quat(rng, da))
    return np.concatenate([q / np.linalg.norm(q), meas[4:7] + rng.normal(size=3) * dt])


def chain_graph(truth, rng, loops=(), dt=0.02, da=0.005):
    """Odometry edges i -> i + 1 with drift noise, plus loop edges (begin, end) measured exactly; the initial poses integrate the odometry."""
    n = truth.shape[0]
    ids, meas = [], []
    for i in range(n - 1):
        ids.append((i, i + 1))
        meas.append(noisy(relative(truth[i], truth[i + 1]), rng, dt, da))
    X = truth.copy()
    for i in range(n - 1):
        X[i + 1, :4] = qmul(X[i, :4], meas[i][:4])
        X[i + 1, 4:7] = X[i, 4:7] + qrot(X[i, :4], meas[i][4:7])
    for a, b in loops:
        ids.append((a, b))
        meas.append(relative(truth[a], truth[b]))
    return X, np.array(ids, np.int32).reshape(-1, 2), np.array(meas).reshape(-1, 7)


_BUILD_DIR = None


def _build(src, name):
    """Compiles tests/cpp/<src> once per process into one temporary directory, removed at exit."""
    global _BUILD_DIR
    if _BUILD_DIR is None:
        _BUILD_DIR = tempfile.mkdtemp(prefix="pose_graph_")
        atexit.register(shutil.rmtree, _BUILD_DIR, True)
    out = os.path.join(_BUILD_DIR, name)
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-w", "-shared", "-fPIC", "-o", out, os.path.join(ROOT, "tests", "cpp", src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return C.CDLL(out)


_ORACLE, _HOST = None, None


def oracle_lib():
    global _ORACLE
    if _ORACLE is None:
        _ORACLE = _build("pg_oracle.cpp", "libpgoracle.so")
    return _ORACLE


def host_lib():
    global _HOST
    if _HOST is None:
        _HOST = _build("pg_host.cpp", "libpghost.so")
    return _HOST


def _p(a):
    return C.c_void_p(a.ctypes.data)


def oracle_optimize(X, ids, meas, W=None, max_iterations=200, ftol=1e-6, ptol=1e-8):
    """The oracle's solve: (poses, initial cost, final cost, iterations, evaluations, termination)."""
    m = ids.shape[0]
    x = np.ascontiguousarray(X, np.float64).copy()
    ids = np.ascontiguousarray(ids, np.int32)
    meas = np.ascontiguousarray(meas, np.float64).reshape(-1, 7)
    Wm = np.ascontiguousarray(np.broadcast_to(np.eye(6) if W is None else W, (m, 6, 6)), np.float64)
    d, i = np.zeros(2), np.zeros(3, np.int32)
    L = oracle_lib()
    L.pgo_optimize(_p(x), x.shape[0], _p(ids), _p(meas), _p(Wm), m, max_iterations, C.c_double(ftol), C.c_double(ptol), _p(d), _p(i))
    return x, d[0], d[1], int(i[0]), int(i[1]), int(i[2])


def oracle_residual(xa, xb, meas, W=None):
    r, Ja, Jb = np.zeros(6), np.zeros((6, 6)), np.zeros((6, 6))
    xa, xb, meas = (np.ascontiguousarray(v, np.float64) for v in (xa, xb, meas))
    Wm = np.ascontiguousarray(np.eye(6) if W is None else W, np.float64)
    oracle_lib().pgo_residual(_p(xa), _p(xb), _p(meas), _p(Wm), _p(r), _p(Ja), _p(Jb))
    return r, Ja, Jb


def oracle_loop_edge(icp_q, icp_t, pose_a, id_a, pose_b, id_b):
    ids, meas = np.zeros(2, np.int32), np.zeros(7)
    a = [np.ascontiguousarray(v, np.float64) for v in (icp_q, icp_t, pose_a, pose_b)]
    oracle_lib().pgo_loop_edge(_p(a[0]), _p(a[1]), _p(a[2]), id_a, _p(a[3]), id_b, _p(ids), _p(meas))
    return (int(ids[0]), int(ids[1])), meas


def oracle_repose(clouds, seg_end, poses_ori, poses_opt, leaf):
    """The oracle's re-posed keyframe clouds: (points [m, 4] float32, counts per keyframe)."""
    c = np.ascontiguousarray(clouds, np.float32).reshape(-1, 4)
    se = np.ascontiguousarray(seg_end, np.int64)
    o, p = np.ascontiguousarray(poses_ori, np.float64), np.ascontiguousarray(poses_opt, np.float64)
    out, cnt = np.zeros((max(c.shape[0], 1), 4), np.float32), np.zeros(se.shape[0], np.int64)
    L = oracle_lib()
    L.pgo_repose.restype = C.c_int
    m = L.pgo_repose(_p(c), _p(se), se.shape[0], _p(o), _p(p), C.c_float(leaf), _p(out), _p(cnt))
    return out[:m].copy(), cnt


def skyline_solve(A, b):
    A, b = np.ascontiguousarray(A, np.float64), np.ascontiguousarray(b, np.float64)
    x = np.zeros_like(b)
    ok = oracle_lib().pgo_skyline_solve(_p(A), _p(b), A.shape[0], _p(x))
    return x if ok else None


def host_solve(N, ids, node_blocks, edge_blocks, rhs):
    """The host build of the device elimination: (x [N, 6], border size, (free nodes, segments, levels))."""
    ids = np.ascontiguousarray(ids, np.int32).reshape(-1, 2)
    ea, eb = np.ascontiguousarray(ids[:, 0]), np.ascontiguousarray(ids[:, 1])
    nb_, eb_, r = (np.ascontiguousarray(v, np.float64) for v in (node_blocks, edge_blocks, rhs))
    x, st = np.zeros((N, 6)), np.zeros(3, np.int32)
    L = host_lib()
    L.pgh_solve.restype = C.c_int
    nb = L.pgh_solve(N, ids.shape[0], _p(ea), _p(eb), _p(nb_), _p(eb_), _p(r), _p(x), _p(st))
    return x, nb, tuple(int(v) for v in st)
