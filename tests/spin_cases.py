"""Constructed inputs of the spinning-lidar front end (ll_spin_*): small clouds that sit on its edges, shared by the oracle and device tests."""
import numpy as np

from loam_livox_b200 import synthetic as S


def ring_points(ring, n, scan_line=16, az0=0.0, az1=-30.0, d=8.0, elev=None):
    """n points of one ring (nominal elevation, or `elev` degrees) from azimuth az0 to az1 (degrees), range d (scalar or [n])."""
    e = np.radians(S.spin_elevations(scan_line)[ring] if elev is None else elev)
    a = np.radians(np.linspace(az0, az1, n)) if n else np.zeros(0)
    d = np.broadcast_to(np.asarray(d, np.float64), (n,))
    return np.c_[d * np.cos(e) * np.cos(a), d * np.cos(e) * np.sin(a), d * np.sin(e) * np.ones(n), np.ones(n)].astype(np.float32)


def interleave(parts):
    """Firing order: point k of every part in turn (the parts' lengths may differ)."""
    out, m = [], max((len(p) for p in parts), default=0)
    for k in range(m):
        out.extend(p[k] for p in parts if k < len(p))
    return np.array(out, np.float32).reshape(-1, 4)


def edge_cases():
    """name -> (scan_line, raw [n, 4])."""
    rng = np.random.default_rng(7)
    cases = {}
    cases["empty_after_filter"] = (16, np.full((3, 4), np.nan, np.float32))
    for n in (1, 4, 5, 6, 11, 12, 13, 24):
        cases[f"kept_{n}"] = (16, interleave([ring_points(r, n // 3 + (1 if r < n % 3 else 0), d=5.0 + r) for r in range(3)]))
    cases["ring_sizes_0_to_13"] = (16, interleave([ring_points(r, r, d=6.0 + 0.1 * r) for r in range(14)] + [ring_points(14, 300, d=rng.uniform(4, 9, 300)),
                                                                                                          ring_points(15, 300, d=7.0)]))
    # ring boundaries of the 16-ring formula: (angle + 15) / 2 + 0.5 integral at -14, 0, 14 degrees, and just either side
    b = []
    for ang in (-14.0, 0.0, 14.0, -16.0, 16.0, 15.0, -15.0):
        for eps in (0.0, 1e-5, -1e-5, 1e-6, -1e-6):
            b.append(ring_points(0, 40, elev=ang + eps, d=rng.uniform(5, 6, 40), az0=rng.uniform(-180, 180), az1=rng.uniform(-180, 180)))
    cases["ring_boundaries_16"] = (16, interleave(b))
    b = []
    for ang in (2.0, -8.83, -24.33, -18.08, -18.33, -17.83, 2.2, -24.5):
        for eps in (0.0, 1e-5, -1e-5, 1e-6, -1e-6):
            b.append(ring_points(0, 40, 64, elev=ang + eps, d=rng.uniform(5, 6, 40), az0=rng.uniform(-180, 180), az1=rng.uniform(-180, 180)))
    cases["ring_boundaries_64"] = (64, interleave(b))
    # sweeps under and over a turn: both endOri corrections, halfPassed at different places
    for sweep in (90.0, 179.9, 180.0, 180.1, 300.0, 359.0, 361.0, 450.0, 540.0, 719.0):
        cases[f"sweep_{sweep:g}"] = (16, S.make_spinning_scan(16, n_azimuth=240, start_azimuth_deg=rng.uniform(-180, 180), sweep_deg=sweep, seed=int(sweep)))
    # occlusions in both directions: a near object in front of a far wall, entered and left
    d = np.full(400, 9.0); d[100:140] = 3.0; d[250:252] = 2.0; d[300:330] = 8.95
    cases["occlusions"] = (16, interleave([ring_points(r, 400, d=d + 0.01 * r, az0=40.0, az1=-40.0) for r in range(16)]))
    # equal curvatures (a plane hit at equal steps: the same sums) and a walk longer than 500 points (no cut in a long smooth ring)
    cases["equal_curvature"] = (16, interleave([ring_points(r, 256, d=4.0, az0=0.0, az1=-25.5) for r in range(16)]))
    cases["long_walk"] = (16, interleave([ring_points(r, 1400, d=10.0 + 0.5 * np.sin(np.linspace(0, 40, 1400)) + (r % 2) * 0.3, az0=170.0, az1=-170.0)
                                          for r in range(16)]))
    # NaN, inf, near and huge points; a curvature that overflows to inf (coordinates of 1e30) and coordinates above 1e36 (removed)
    raw = S.make_spinning_scan(16, n_azimuth=200, seed=3, nan_frac=0.05, near_frac=0.05)
    raw[5, 0] = np.inf; raw[9, 2] = -np.inf; raw[17, :3] = 1e-3; raw[30, :3] = [1e30, 1e30, 0.0]; raw[40, :3] = [2e36, 1.0, 0.0]; raw[41, :3] = [1e35, -1e35, 0.0]
    cases["nan_inf_near_huge"] = (16, raw)
    # a noisy scan: many sharp candidates per sub-scan (the 20 / 200 caps) and few flat ones
    cases["noisy_caps"] = (16, S.make_spinning_scan(16, n_azimuth=1200, seed=11, range_sigma=0.08))
    cases["noisy_caps_64"] = (64, S.make_spinning_scan(64, n_azimuth=600, seed=12, range_sigma=0.08))
    # rising range with alternating steps at 100 m: every gap is a cut but none trips the parallel-beam test, so sub-scans reach the caps
    for inc in (1.6, 3.0):
        k = np.arange(1300)
        d = 100 + inc * (k // 2) + (k % 2) * inc * 0.5
        cases[f"sharp_caps_{inc:g}"] = (16, interleave([ring_points(r, 1300, d=d, az0=130.0, az1=-130.0) for r in range(16)]))
    return cases
