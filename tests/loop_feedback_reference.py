"""Loop feedback restated (DESIGN.md §4.6.2), bit for bit: ll_loop_correction's rule in Python floats (its libm calls through the math module,
the same C library functions), the pose composition with the library's association (quat_mul, exact_math.cuh qrot_d), and the window
correction kernel's fp64 transform of float points in NumPy.  Also a reader of a version-3 loop image's FEEDBACK section."""
import math
import struct

import numpy as np

IDENTITY = ((1.0, 0.0, 0.0, 0.0), (0.0, 0.0, 0.0))


def qmul(a, b):
    """quat_mul: each component summed left to right as written."""
    return (a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
            a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
            a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1],
            a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0])


def qrot(q, v):
    """qrot_d on one fp64 vector: uv = 2 (u x v); v + w uv + u x uv."""
    w, ux, uy, uz = q
    cx, cy, cz = uy * v[2] - uz * v[1], uz * v[0] - ux * v[2], ux * v[1] - uy * v[0]
    cx, cy, cz = cx + cx, cy + cy, cz + cz
    dx, dy, dz = uy * cz - uz * cy, uz * cx - ux * cz, ux * cy - uy * cx
    return ((v[0] + cx * w) + dx, (v[1] + cy * w) + dy, (v[2] + cz * w) + dz)


def compose(a, b):
    """a o b = (q_a q_b, R_a t_b + t_a)."""
    r = qrot(a[0], b[1])
    return qmul(a[0], b[0]), tuple(r[k] + a[1][k] for k in range(3))


def inverse(a):
    qc = (a[0][0], -a[0][1], -a[0][2], -a[0][3])
    r = qrot(qc, a[1])
    return qc, tuple(-x for x in r)


def pose(row):
    """a [7] row (q w, x, y, z, t) as a pose"""
    return tuple(float(x) for x in row[:4]), tuple(float(x) for x in row[4:7])


def keyframe_correction(ori, opt, k):
    return IDENTITY if k == 0 else compose(pose(opt[k]), inverse(pose(ori[k])))


def correction(ori, opt, f, s):
    """ll_loop_correction: A_0 up to f[0], A_(n-1) from f[n - 1], A_k at f[k], the slerp (shorter arc) and lerp in between."""
    n = len(f)
    if s <= f[0]:
        return IDENTITY
    if s >= f[n - 1]:
        return keyframe_correction(ori, opt, n - 1)
    k = max(j for j in range(n) if f[j] <= s)
    a = keyframe_correction(ori, opt, k)
    if s == f[k]:
        return a
    b = keyframe_correction(ori, opt, k + 1)
    u = float(s - f[k]) / float(f[k + 1] - f[k])
    dot = 0.0
    for j in range(4):
        dot = dot + a[0][j] * b[0][j]
    qb = [-x if dot < 0 else x for x in b[0]]
    dn = sn = 0.0
    for j in range(4):
        x, y = a[0][j] - qb[j], a[0][j] + qb[j]
        dn, sn = dn + x * x, sn + y * y
    theta = 2.0 * math.atan2(math.sqrt(dn), math.sqrt(sn))
    if theta == 0.0:
        q = a[0]
    else:
        st = math.sin(theta)
        wa, wb = math.sin((1.0 - u) * theta) / st, math.sin(u * theta) / st
        q = tuple(wa * a[0][j] + wb * qb[j] for j in range(4))
    return q, tuple(a[1][j] + u * (b[1][j] - a[1][j]) for j in range(3))


def segment_delta(ori, opt, f, n, prev_opt, n_prev, s):
    """A(s) o A_prev(s)^-1 of a window segment at frame index s (n_prev 0: the identity before the first loop)."""
    a = correction(ori[:n], opt[:n], f[:n], s)
    b = correction(ori[:n_prev], prev_opt[:n_prev], f[:n_prev], s) if n_prev else IDENTITY
    return compose(a, inverse(b))


def transform(pts, d):
    """the correction kernel on float32 [n, 4] points: fp64 qrot_d, + t, rounded once to float; intensity kept."""
    q, t = d
    p = pts[:, :3].astype(np.float64)
    r = qrot(q, (p[:, 0], p[:, 1], p[:, 2]))
    out = pts.copy()
    for k in range(3):
        out[:, k] = (r[k] + t[k]).astype(np.float32)
    return out


def feedback_section(image):
    """A version-3 loop image's FEEDBACK section: (n_applied, C, f[n_keyframes], frame[n_segments])."""
    off = struct.unpack_from("<Q", image, 24 + 16 * 13)[0]
    na = struct.unpack_from("<i", image, off + 4)[0]
    c = struct.unpack_from("<7d", image, off + 8)
    nk, ns = struct.unpack_from("<qq", image, off + 64)
    f = np.frombuffer(image, "<i4", nk, off + 80)
    fr = np.frombuffer(image, "<i4", ns, off + 80 + 4 * nk)
    return na, (tuple(c[:4]), tuple(c[4:])), f.copy(), fr.copy()


def history(mapper_image, c):
    """a mapper image's history window of class c (0 corner, 1 surface): segment sizes and float32 [n, 4] points"""
    off, _ = struct.unpack_from("<QQ", mapper_image, 24 + 16 * (2 + c))
    ns, npts = struct.unpack_from("<qq", mapper_image, off)
    sizes = np.frombuffer(mapper_image, "<i4", ns, off + 16)
    pts = np.frombuffer(mapper_image, "<f4", 4 * npts, off + 16 + 4 * ns).reshape(npts, 4)
    return sizes.copy(), pts.copy()


def corrected_history(sizes, pts, deltas):
    """every segment of a window through the transform with its own delta"""
    out, o = [], 0
    for z, d in zip(sizes, deltas):
        out.append(transform(pts[o:o + z], d))
        o += z
    return np.concatenate(out) if out else pts[:0].copy()
