"""Extended-precision reference of the solver's evaluation: residuals, tangent-space Jacobians, Huber weights, the loss-corrected normal
equations, the cost and the per-block L1 norms of the residual blocks of one ICP iteration -- NumPy only, in np.longdouble.

Restated from the published behaviour of the pieces the reference registration uses (see oracle/orc_solver.hpp and csrc/solve.cu for the line
citations), independently of both the library's closed form and the oracle's Jets:

- residual functors of ceres_icp.hpp: point-to-line r = d - (d.v) v, point-to-plane r = (d.v) v, with d = q_last (q p + t) + t_last - a; the
  *_mb forms replace (q, t) by (Identity.slerp(s, q), s t) with Eigen's slerp (plain lerp when |w| >= 1 - eps, eps = 2^-52; scale1 negated
  when w < 0; the result is not re-normalised);
- ceres::EigenQuaternionParameterization::Plus(x, delta) = [sin|delta| / |delta| delta, cos|delta|] * q (quaternion product);
- ceres::HuberLoss(a) with the Corrector: since rho'' <= 0 the weight on J^T J and J^T r is rho', the cost is rho / 2 and the L1 norm of a block
  is || sqrt(rho') r ||_1.

The Jacobian is taken by COMPLEX STEP through Plus(x, delta) at delta = 0 in np.clongdouble: every functor is analytic in x (branches are taken
on the real part), so Im f(Plus(x, i h e_c)) / h is the derivative of the expression as written, exact to working precision for h = 1e-300.
Sums run in np.longdouble (64-bit significand or more).

Each output also comes with an a-priori rounding scale S: a bound, up to a small constant, on how much fp64 arithmetic of ANY correct formula
of the same quantity can differ from the exact value per unit roundoff.  See `normal_equations` for its definition.
"""
from __future__ import annotations

import numpy as np

LD = np.longdouble
CLD = np.clongdouble
EXTENDED = np.finfo(LD).nmant >= 63   # x86 80-bit (63) or IEEE quad (112); the tests skip where long double is plain double
EPS64 = 2.0 ** -53                    # unit roundoff of fp64
H_STEP = LD("1e-300")                 # complex step: h^2 vanishes against 1 even in long double


def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def _rot(q, v):
    """q (w, x, y, z) applied to v: v + 2 w (u x v) + 2 u x (u x v) (Eigen's _transformVector; for a non-unit q, as Eigen computes it)."""
    w, u = q[0], q[1:]
    c = _cross(u, v)
    c = (2 * c[0], 2 * c[1], 2 * c[2])
    e = _cross(u, c)
    return (v[0] + w * c[0] + e[0], v[1] + w * c[1] + e[1], v[2] + w * c[2] + e[2])


def _qmul(a, b):
    aw, ax, ay, az = a
    bw, bx, by, bz = b
    return (aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
            aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw)


def plus(x, delta, dtype=CLD):
    """EigenQuaternionParameterization::Plus (no box projection: the bounds are not part of the manifold).  x = (qx, qy, qz, qw, tx, ty, tz).
    sin|d| / |d| and cos|d| as their power series in z = d.d (analytic in d; exact here because |z| <= 1e-12 wherever it is used)."""
    d = [dtype(v) for v in delta]
    z = d[0] * d[0] + d[1] * d[1] + d[2] * d[2]
    assert abs(complex(z)) <= 1e-12
    sinc = 1 - z / 6 + z * z / 120
    cosn = 1 - z / 2 + z * z / 24
    q = (dtype(x[3]), dtype(x[0]), dtype(x[1]), dtype(x[2]))
    qn = _qmul((cosn, sinc * d[0], sinc * d[1], sinc * d[2]), q)
    return qn, tuple(dtype(x[4 + k]) + d[3 + k] for k in range(3))


def _slerp_scales(w, s, dtype):
    """Eigen Quaternion::slerp(s, other) from Identity: (scale0, scale1) with scale1 already sign-flipped for w < 0.  Branches on Re(w)."""
    wr = float(np.real(w)) if dtype in (CLD, np.complex128) else float(w)
    absd = w if wr >= 0 else -w
    if abs(wr) >= 1.0 - 2.0 ** -52:
        sc0, sc1 = 1 - s, s
    else:
        th = np.arccos(absd)
        st = np.sin(th)
        sc0, sc1 = np.sin((1 - s) * th) / st, np.sin(s * th) / st
    if wr < 0:
        sc1 = -sc1
    return sc0, sc1


def _chain(B, q, t, q_last, t_last, dtype):
    """pt_tr = q_last (q' p + t') + t_last with (q', t') = (q, t) or the slerp / scaled pair of the *_mb functors; returns (pt_tr, q' p)."""
    p = tuple(B[:, 1 + k].astype(dtype) for k in range(3))
    s = B[:, 10]
    mb = ~np.isnan(s)
    if mb.any():
        sd = np.where(mb, s, 1.0).astype(dtype)
        sc0, sc1 = _slerp_scales(q[0], sd, dtype)
        qi = (np.where(mb, sc0 + sc1 * q[0], q[0]), np.where(mb, sc1 * q[1], q[1]), np.where(mb, sc1 * q[2], q[2]), np.where(mb, sc1 * q[3], q[3]))
        ti = tuple(np.where(mb, sd * t[k], t[k]) for k in range(3))
    else:
        qi, ti = q, t
    y = _rot(qi, p)
    ql = tuple(dtype(v) for v in q_last)
    w = _rot(ql, tuple(y[k] + ti[k] for k in range(3)))
    return tuple(w[k] + dtype(t_last[k]) for k in range(3)), y


def residuals(B, q_last, t_last, q, t, dtype=LD):
    """r (M x 3) and pt_tr (M x 3), y = q' p (M x 3) of the blocks B (oracle layout: type 0 line / 1 plane, p, a, v, s or NaN)."""
    pt, y = _chain(B, q, t, q_last, t_last, dtype)
    d = tuple(pt[k] - B[:, 4 + k].astype(dtype) for k in range(3))
    v = tuple(B[:, 7 + k].astype(dtype) for k in range(3))
    dv = d[0] * v[0] + d[1] * v[1] + d[2] * v[2]
    line = B[:, 0] == 0
    r = tuple(np.where(line, d[k] - dv * v[k], dv * v[k]) for k in range(3))
    return np.stack(r, 1), np.stack(pt, 1), np.stack(y, 1)


def jacobians(B, q_last, t_last, x, dtype=CLD, h=H_STEP):
    """Residuals r (M x 3), tangent Jacobians J (M x 3 x 6) of r and G (M x 3 x 6) of pt_tr, and y, by complex step through Plus(x, i h e_c)."""
    M = B.shape[0]
    J = np.zeros((M, 3, 6), np.longdouble if dtype == CLD else np.float64)
    G = np.zeros_like(J)
    r0 = y0 = None
    for c in range(6):
        delta = [0, 0, 0, 0, 0, 0]
        delta[c] = dtype(1j * h)
        q, t = plus(x, delta, dtype)
        r, pt, y = residuals(B, q_last, t_last, q, t, dtype)
        J[:, :, c] = r.imag / h
        G[:, :, c] = pt.imag / h
        if c == 0:
            r0, y0 = r.real, y.real
    return r0, J, G, y0


def huber(sq, a):
    """(rho, rho') of ceres::HuberLoss(a) at s = |r|^2 (rho' floored at DBL_MIN as Ceres does)."""
    a = LD(a)
    b = a * a
    r = np.sqrt(sq)
    tail = sq > b
    rho = np.where(tail, 2 * a * r - b, sq)
    rho1 = np.where(tail, np.maximum(LD(np.finfo(np.float64).tiny), a / np.where(r > 0, r, 1)), LD(1))
    return rho, rho1, tail


def normal_equations(B, q_last, t_last, x, huber_a, mult=None, h=H_STEP, dtype=CLD):
    """Loss-corrected J^T J (6 x 6), J^T r (6), cost, per-block L1 norms, and their rounding scales.

    B: M x 11 blocks (oracle layout); mult: optional per-block multiplicity (a block repeated k times contributes k times -- lets the tests
    reference 400k-slot problems built from a few thousand distinct blocks).

    Rounding scales.  Per block, with u = 2^-53, G the Jacobian of pt_tr (before the projection), n = |v|^2, f = (1 + n)^2 (|J| <= (1 + n)|G|
    for lines and n |G| for planes), A = |a| + |t_last| + |q' p| + |t'| (the magnitudes that cancel in d = pt_tr - a), tail = |r|^2 > a^2:
      S_H[i,j] = sum rho' f |G_i| |G_j| (1 + tail (1 + n) A / |r|)   -- the closed form subtracts |v|^2 beta beta^T from G^T G, so its rounding
                                                                     scales with the unprojected columns; in the Huber tail rho' = a / |r|
                                                                     inherits the relative error of |r|
      S_g[j]   = sum rho' f |G_j| (|r| + A)
      S_cost   = sum rho' f |r| (|r| + A)
      S_l1     = sqrt(rho') (1 + n) 3 (|r| + A)                     (per block)
    Any fp64 evaluation whose per-block formula has a rounding chain of depth d1 and whose sums have depth d2 differs from the exact value by
    at most about (d1 + d2) u S; the tests state their constant K against that.
    """
    B = np.ascontiguousarray(B, np.float64)
    M = B.shape[0]
    w = np.ones(M, np.longdouble) if mult is None else np.asarray(mult).astype(np.longdouble)
    r, J, G, y = jacobians(B, q_last, t_last, x, dtype, h)
    sq = (r * r).sum(1)
    rho, rho1, tail = huber(sq, huber_a)
    rn = np.sqrt(sq)
    sc = np.sqrt(rho1)
    l1 = np.abs(sc[:, None] * r).sum(1)
    Hm = np.einsum("m,mki,mkj->ij", w * rho1, J, J)
    g = np.einsum("m,mki,mk->i", w * rho1, J, r)
    cost = (w * rho / 2).sum()
    n = (B[:, 7:10].astype(np.longdouble) ** 2).sum(1)
    f = (1 + n) ** 2
    tl = np.asarray(t_last, np.longdouble)
    A = (np.sqrt((B[:, 4:7].astype(np.longdouble) ** 2).sum(1)) + np.sqrt((tl ** 2).sum()) + np.sqrt((y ** 2).sum(1))
         + np.sqrt((np.asarray(x[4:7], np.longdouble) ** 2).sum()) * np.where(np.isnan(B[:, 10]), 1, np.abs(np.nan_to_num(B[:, 10]))))
    Gn = np.sqrt((G * G).sum(1))                                               # M x 6 column norms
    hf = 1 + np.where(tail, (1 + n) * A / np.where(rn > 0, rn, 1), 0)
    S_H = np.einsum("m,mi,mj->ij", w * rho1 * f * hf, Gn, Gn)
    S_g = np.einsum("m,mi->i", w * rho1 * f * (rn + A), Gn)
    S_c = (w * rho1 * f * rn * (rn + A)).sum()
    S_l1 = sc * (1 + n) * 3 * (rn + A)
    return dict(H=Hm, g=g, cost=cost, l1=l1, r=r, J=J, rho1=rho1, S_H=S_H, S_g=S_g, S_cost=S_c, S_l1=S_l1, n=w.sum())


def quat_axis_angle(axis, angle):
    """Unit quaternion (w, x, y, z) of a rotation by `angle` about `axis`."""
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    return np.concatenate([[np.cos(angle / 2)], np.sin(angle / 2) * a])


def qrot64(q, v):
    """fp64 rotation of the rows of v by q (w, x, y, z): test-data construction only."""
    w, u = q[0], np.asarray(q[1:])
    c = 2 * np.cross(u, v)
    return v + w * c + np.cross(u, c)


def make_blocks(M, rng, kind="mix", q_last=(1, 0, 0, 0), t_last=(0, 0, 0), radius=30.0, vnorm=1.0, offset=(0.0, 0.3), blur=None, true_x=None):
    """M residual blocks in the oracle's layout (type 0 line / 1 plane, p, a, v, s or NaN) around a true increment `true_x`: features p
    (scan frame, fp32) within `radius` m, anchors a (fp32) on the line / plane through the true world point, off it by a distance drawn
    from `offset`, directions / normals of length `vnorm`.  kind: 'line', 'plane' or 'mix' (alternating)."""
    p = rng.uniform(-1, 1, (M, 3)) * radius
    p = p.astype(np.float32).astype(np.float64)
    tx = np.array([0, 0, 0, 1, 0, 0, 0.0]) if true_x is None else np.asarray(true_x, np.float64)
    qi = np.array([tx[3], tx[0], tx[1], tx[2]])
    pw = qrot64(np.asarray(q_last, np.float64), qrot64(qi, p) + tx[4:7]) + np.asarray(t_last, np.float64)
    v = rng.normal(size=(M, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    typ = {"line": np.zeros(M), "plane": np.ones(M), "mix": np.arange(M) % 2}[kind]
    perp = np.cross(v, rng.normal(size=(M, 3)))
    perp /= np.linalg.norm(perp, axis=1, keepdims=True)
    off = rng.uniform(*offset, M)
    along = rng.uniform(-2, 2, M)
    a = np.where(typ[:, None] == 0, pw + along[:, None] * v + off[:, None] * perp, pw + along[:, None] * perp + off[:, None] * v)
    a = a.astype(np.float32).astype(np.float64)
    s = np.full(M, np.nan) if blur is None else np.broadcast_to(np.asarray(blur, np.float32).astype(np.float64), (M,)).copy()
    return np.column_stack([typ, p, a, v * vnorm, s])


def upper(Hm):
    """The 21 upper-triangular entries, row-major (the library's out28 order)."""
    return np.array([Hm[i, j] for i in range(6) for j in range(i, 6)])
