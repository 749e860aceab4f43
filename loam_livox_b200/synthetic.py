"""Seeded synthetic Livox Mid-40 scans, maps and trajectories (SURVEY.md §8d).

The reference ships no data, fixtures or tests (SURVEY.md §4), so every input used by tests/ and bench.py is
generated here: an analytic room (floor, ceiling, four walls) with 24 square pillars, a rosette-scanning
sensor model whose x axis looks forward (the extractor assumes that:
loam_livox/source/livox_feature_extractor.hpp:518), closed-form ray casting, and world-frame feature
maps sampled directly from the scene geometry.  NumPy only; everything is a pure function of its seed.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

SEED = 20260922

# ------------------------------------------------------------------ scene
ROOM_LO = np.array([-2.0, -6.0, -1.5])
ROOM_HI = np.array([40.0, 6.0, 3.0])
PILLAR_HALF = 0.2
PILLAR_XS = [5.0 + 4.0 * i for i in range(8)]
PILLAR_YS = [-3.7, 0.9, 3.9]
PILLARS = [(x, y) for x in PILLAR_XS for y in PILLAR_YS]  # 24 pillars, floor to ceiling


def quat_mul(a, b):
    """Hamilton product, (w,x,y,z)."""
    aw, ax, ay, az = a
    bw, bx, by, bz = b
    return np.array([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                     aw * by + ay * bw + az * bx - ax * bz, aw * bz + az * bw + ax * by - ay * bx])


def quat_from_euler(roll, pitch, yaw):
    cr, sr, cp, sp, cy, sy = math.cos(roll / 2), math.sin(roll / 2), math.cos(pitch / 2), math.sin(pitch / 2), math.cos(yaw / 2), math.sin(yaw / 2)
    return np.array([cr * cp * cy + sr * sp * sy, sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy])


def quat_to_mat(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def quat_angle(a, b):
    d = abs(float(np.dot(a, b)))
    return 2.0 * math.acos(min(1.0, d))


def raycast(origin, dirs):
    """First hit distance of rays origin + s*dirs (dirs: [n,3], unit) with the room interior and the pillars."""
    n = dirs.shape[0]
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / dirs
        # room: we are inside the box, take the exit distance
        t1 = (ROOM_LO - origin) * inv
        t2 = (ROOM_HI - origin) * inv
        t_exit = np.nanmin(np.maximum(t1, t2), axis=1)
        best = t_exit
        for (px, py) in PILLARS:
            lo = np.array([px - PILLAR_HALF, py - PILLAR_HALF, ROOM_LO[2]])
            hi = np.array([px + PILLAR_HALF, py + PILLAR_HALF, ROOM_HI[2]])
            a = (lo - origin) * inv
            b = (hi - origin) * inv
            tn = np.nanmax(np.minimum(a, b), axis=1)
            tf = np.nanmin(np.maximum(a, b), axis=1)
            hit = (tn <= tf) & (tn > 1e-6)
            best = np.where(hit & (tn < best), tn, best)
    assert best.shape == (n,)
    return best


def rosette(n, petals=20, half_fov_deg=19.2, f_rot=0.317):
    """(y/x, z/x) image-plane coordinates of a Mid-40 style rosette sampled at n points over one frame."""
    u = np.arange(n, dtype=np.float64) / n
    rho = math.tan(math.radians(half_fov_deg)) * np.abs(np.sin(math.pi * petals * u))
    psi = 2.0 * math.pi * (petals * f_rot) * u
    return rho * np.cos(psi), rho * np.sin(psi)


@dataclass
class Pose:
    q: np.ndarray  # (w,x,y,z)
    t: np.ndarray

    def R(self):
        return quat_to_mat(self.q)


def default_pose():
    return Pose(quat_from_euler(0.01, -0.02, 0.05), np.array([0.3, 0.2, 0.1]))


def perturb_pose(pose, rng, dt=0.1, dang_deg=2.0):
    d = rng.uniform(-dt, dt, 3)
    e = np.radians(rng.uniform(-dang_deg, dang_deg, 3))
    return Pose(quat_mul(pose.q, quat_from_euler(*e)), pose.t + d)


def make_scan(n, pose=None, seed=SEED, range_sigma=0.004, zero_frac=0.005, nan_frac=0.001, low_refl_frac=0.003, yaw_offset_deg=0.0):
    """One raw sensor-frame scan: float32 [n,4] = x,y,z,reflectivity, with zero returns and NaNs mixed in."""
    pose = pose or default_pose()
    rng = np.random.default_rng(seed)
    iy, iz = rosette(n)
    d = np.stack([np.ones(n), iy, iz], axis=1)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    if yaw_offset_deg:
        Rz = quat_to_mat(quat_from_euler(0, 0, math.radians(yaw_offset_deg)))
        d_s = d @ Rz.T
    else:
        d_s = d
    dw = d_s @ pose.R().T
    rng_true = raycast(pose.t, dw)
    r = rng_true + rng.normal(0.0, range_sigma, n)
    pts = d_s * r[:, None]
    inten = rng.uniform(20.0, 150.0, n)
    low = rng.random(n) < low_refl_frac
    inten[low] = rng.uniform(0.0, 5e-5, int(low.sum()))
    out = np.concatenate([pts, inten[:, None]], axis=1).astype(np.float32)
    zero = rng.random(n) < zero_frac
    nan = rng.random(n) < nan_frac
    zero[0] = False
    nan[0] = False
    out[zero, :3] = 0.0
    out[nan, :3] = np.nan
    return out


def make_triple_scan(n_total, pose=None, seed=SEED):
    """Mid-100 style frame: three Mid-40 heads yawed -25/0/+25 degrees, concatenated
    (loam_livox/source/laser_feature_extractor.hpp:353-358 sums the per-lidar feature clouds)."""
    n = n_total // 3
    return [make_scan(n, pose, seed + k, yaw_offset_deg=y) for k, y in enumerate((-25.0, 0.0, 25.0))]


# ------------------------------------------------------------------ maps
def _surfaces():
    """List of (origin, edge_u, edge_v, normal) rectangles: room faces + pillar faces."""
    lo, hi = ROOM_LO, ROOM_HI
    rects = []
    ext = hi - lo
    for ax in range(3):
        u_ax, v_ax = [a for a in range(3) if a != ax]
        for side, val in ((0, lo[ax]), (1, hi[ax])):
            o = lo.copy()
            o[ax] = val
            eu = np.zeros(3); eu[u_ax] = ext[u_ax]
            ev = np.zeros(3); ev[v_ax] = ext[v_ax]
            nrm = np.zeros(3); nrm[ax] = 1.0 if side == 0 else -1.0
            rects.append((o, eu, ev, nrm))
    h = ROOM_HI[2] - ROOM_LO[2]
    for (px, py) in PILLARS:
        for ax, sgn in ((0, -1), (0, 1), (1, -1), (1, 1)):
            o = np.array([px - PILLAR_HALF, py - PILLAR_HALF, ROOM_LO[2]])
            nrm = np.zeros(3); nrm[ax] = sgn
            if sgn > 0:
                o[ax] += 2 * PILLAR_HALF
            eu = np.zeros(3); eu[1 - ax] = 2 * PILLAR_HALF
            ev = np.array([0.0, 0.0, h])
            rects.append((o, eu, ev, nrm))
    return rects


def _edges():
    """Line segments (p0, p1): pillar vertical edges and the 12 room edges."""
    segs = []
    for (px, py) in PILLARS:
        for sx in (-1, 1):
            for sy in (-1, 1):
                x, y = px + sx * PILLAR_HALF, py + sy * PILLAR_HALF
                segs.append((np.array([x, y, ROOM_LO[2]]), np.array([x, y, ROOM_HI[2]])))
    lo, hi = ROOM_LO, ROOM_HI
    c = [np.array([x, y, z]) for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])]
    for i in range(8):
        for j in range(i + 1, 8):
            if np.count_nonzero(c[i] != c[j]) == 1:
                segs.append((c[i], c[j]))
    return segs


def make_map(n_corner, n_surf, seed=SEED, surf_sigma=0.002, corner_sigma=0.0):
    """World-frame feature maps sampled directly from the scene: float32 [n,4] (intensity = 0)."""
    rng = np.random.default_rng(seed + 1)
    rects = _surfaces()
    areas = np.array([np.linalg.norm(np.cross(eu, ev)) for (_, eu, ev, _) in rects])
    counts = rng.multinomial(n_surf, areas / areas.sum())
    chunks = []
    for (o, eu, ev, nrm), k in zip(rects, counts):
        a = rng.random((k, 1)); b = rng.random((k, 1))
        p = o + a * eu + b * ev + nrm * rng.normal(0.0, surf_sigma, (k, 1))
        chunks.append(p)
    surf = np.concatenate(chunks, axis=0)
    surf = surf[rng.permutation(surf.shape[0])]
    segs = _edges()
    lens = np.array([np.linalg.norm(b - a) for a, b in segs])
    counts = rng.multinomial(n_corner, lens / lens.sum())
    chunks = []
    for (a, b), k in zip(segs, counts):
        s = rng.random((k, 1))
        p = a + s * (b - a)
        if corner_sigma > 0:
            p = p + rng.normal(0.0, corner_sigma, (k, 3))
        chunks.append(p)
    corner = np.concatenate(chunks, axis=0)
    corner = corner[rng.permutation(corner.shape[0])]
    z = lambda p: np.concatenate([p, np.zeros((p.shape[0], 1))], axis=1).astype(np.float32)
    return z(corner), z(surf)


def make_features(n_corner, n_surf, pose=None, seed=SEED, sigma=0.004, max_range=25.0):
    """Sensor-frame corner / surface feature clouds sampled directly from the scene inside the sensor's FOV
    (registration-only mode: features given, no extractor).  intensity carries a fake timestamp in [0, 0.1]."""
    pose = pose or default_pose()
    rng = np.random.default_rng(seed + 2)
    R, t = pose.R(), pose.t
    cos_fov = math.cos(math.radians(19.2))

    def in_fov(pw):
        ps = (pw - t) @ R
        rn = np.linalg.norm(ps, axis=1)
        ok = (ps[:, 0] > 0.5) & (ps[:, 0] / np.maximum(rn, 1e-9) > cos_fov) & (rn < max_range)
        return ps, ok

    def collect(sampler, n):
        got = []
        tot = 0
        while tot < n:
            pw = sampler(max(4 * n, 100000))
            ps, ok = in_fov(pw)
            ps = ps[ok]
            got.append(ps)
            tot += ps.shape[0]
        ps = np.concatenate(got, axis=0)[:n]
        ps = ps + rng.normal(0.0, sigma, ps.shape)
        ts = rng.uniform(0.0, 0.1, (ps.shape[0], 1))
        return np.concatenate([ps, ts], axis=1).astype(np.float32)

    def surf_sampler(m):
        c, s = make_map(1, m, seed=int(rng.integers(1 << 30)), surf_sigma=0.0)
        return s[:, :3].astype(np.float64)

    def corner_sampler(m):
        c, s = make_map(m, 1, seed=int(rng.integers(1 << 30)))
        return c[:, :3].astype(np.float64)

    return collect(corner_sampler, n_corner), collect(surf_sampler, n_surf)


def make_distorted_features(pose_last, pose_curr, nc, ns, seed=0):
    """Features of a scan taken WHILE the sensor moves from pose_last to pose_curr: the point with time fraction s is seen from
    pose_last * (slerp(I, s, q_inc), s t_inc) -- the motion model the *_mb functors assume.  intensity = time stamp in [0, 0.1]."""
    from scipy.spatial.transform import Rotation as Rsc, Slerp
    fc, fs = make_features(nc, ns, pose_curr, seed=SEED + seed)
    Rl, Rc = pose_last.R(), pose_curr.R()
    R_inc = Rl.T @ Rc
    t_inc = Rl.T @ (pose_curr.t - pose_last.t)
    sl = Slerp([0.0, 1.0], Rsc.from_matrix(np.stack([np.eye(3), R_inc])))
    out = []
    for f in (fc, fs):
        s = f[:, 3].astype(np.float64) / 0.1
        pw = f[:, :3].astype(np.float64) @ Rc.T + pose_curr.t                 # world points (sampled from the scene at pose_curr)
        Ri = sl(s).as_matrix()                                                # interpolated increment per point
        y = (pw - pose_last.t) @ Rl - s[:, None] * t_inc                      # q_last^-1 (pw - t_last) - s t_inc
        ps = np.einsum("nji,nj->ni", Ri, y)                                   # R_i^T y
        g = f.copy(); g[:, :3] = ps.astype(np.float32)
        out.append(g)
    return out[0], out[1]


def trajectory(n_scans=1000, n_static=50, dt=0.1, speed=1.0, yaw_rate_deg=5.0, zero_mean_yaw=False, y0=0.2):
    """C3 trajectory: n_static stationary scans, then forward motion with sinusoidal yaw (SURVEY.md §8d)."""
    poses = []
    x, y, yaw = 0.3, y0, 0.0   # y0: the pillar rows stand at y = -3.7, 0.9, 3.9 (+-0.2); a 1000-scan path must stay in the aisle between them
    for i in range(n_scans):
        if i >= n_static:
            k = i - n_static
            # zero_mean_yaw: a cosine rate, so that the yaw itself is a zero-mean sinusoid.  The default sine rate integrates to a one-sided yaw and walks the
            # sensor through the side wall after ~700 scans (found when config C3 was first run at its full 1000 scans); short test sequences keep it.
            ph = 2 * math.pi * k * dt / 20.0
            yaw_rate = math.radians(yaw_rate_deg) * (math.cos(ph) if zero_mean_yaw else math.sin(ph))
            yaw += yaw_rate * dt
            x += speed * dt * math.cos(yaw) * 0.3  # keep inside the 42 m room over 950 steps
            y += speed * dt * math.sin(yaw) * 0.3
        poses.append(Pose(quat_from_euler(0.0, 0.0, yaw), np.array([x, y, 0.1])))
    return poses
