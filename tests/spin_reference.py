"""An independent NumPy restatement of the reference's Velodyne front end (laser_feature_extractor.hpp:393-825), float32 with the written
association, for checking the oracle (oracle/orc_spin.hpp).  It uses the closed forms the device uses where the oracle keeps the literal
loops: picked = beam(k) OR any backward occlusion of i = k ... k + 5, and a stable sort of each sub-scan in place of the insertion sort."""
import math

import numpy as np

F = np.float32
PI = math.pi


def _ori(x, y):
    return F(-F(math.atan2(float(y), float(x))))


def extract(raw, scan_line=16, minimum_range=0.1, plane_resolution=0.4, voxel_grid=None):
    raw = np.asarray(raw, np.float32).reshape(-1, 4)
    with np.errstate(over="ignore", invalid="ignore"):
        fin = np.isfinite(raw[:, :3]).all(1) & (np.abs(raw[:, :3]) <= F(1e36)).all(1)
        x, y, z = raw[:, 0], raw[:, 1], raw[:, 2]
        r2 = x * x + y * y + z * z
        thr = F(minimum_range)
        keep = fin & ~(r2 < thr * thr)
    pts = raw[keep]
    scans = [[] for _ in range(scan_line)]
    if len(pts):
        so = _ori(pts[0, 0], pts[0, 1])
        eo = F(float(_ori(pts[-1, 0], pts[-1, 1])) + 2 * PI)
        if float(F(eo - so)) > 3 * PI:
            eo = F(float(eo) - 2 * PI)
        elif float(F(eo - so)) < PI:
            eo = F(float(eo) + 2 * PI)
        half = False
        for p in pts:
            px, py, pz = F(p[0]), F(p[1]), F(p[2])
            with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
                t = F(math.atan(float(F(pz / np.sqrt(F(px * px + py * py))))))
            angle = F(float(F(t * F(180))) / PI)
            if scan_line == 16:
                sid = int(float(F(F(angle + F(15)) / F(2))) + 0.5)
                if sid > 15 or sid < 0:
                    continue
            else:
                a = float(angle)
                sid = int(float(F(F(2) - angle)) * 3.0 + 0.5) if a >= -8.83 else 32 + int((-8.83 - a) * 2.0 + 0.5)
                if angle > F(2) or a < -24.33 or sid > 50 or sid < 0:
                    continue
            o = _ori(px, py)
            if not half:
                if float(o) < float(so) - PI / 2:
                    o = F(float(o) + 2 * PI)
                elif float(o) > float(so) + PI * 3 / 2:
                    o = F(float(o) - 2 * PI)
                half = float(F(o - so)) > PI
            else:
                o = F(float(o) + 2 * PI)
                if float(o) < float(eo) - PI * 3 / 2:
                    o = F(float(o) + 2 * PI)
                elif float(o) > float(eo) + PI / 2:
                    o = F(float(o) - 2 * PI)
            rel = F(F(o - so) / F(eo - so))
            scans[sid].append([px, py, pz, F(sid + 0.1 * float(rel))])
    start, end, ring, cloud = [], [], [], []
    for r in range(scan_line):
        start.append(len(cloud) + 5)
        cloud += scans[r]
        ring += [r] * len(scans[r])
        end.append(len(cloud) - 6)
    c = np.array(cloud, np.float32).reshape(-1, 4)
    N = len(c)
    curv, occl, beam = np.zeros(N, F), np.zeros(N, bool), np.zeros(N, bool)
    with np.errstate(over="ignore", invalid="ignore"):
        for i in range(5, N - 5):
            d = [F(0)] * 3
            for ax in range(3):
                s = c[i - 5, ax]
                for k in (i - 4, i - 3, i - 2, i - 1):
                    s = F(s + c[k, ax])
                s = F(s - F(F(10) * c[i, ax]))
                for k in range(i + 1, i + 6):
                    s = F(s + c[k, ax])
                d[ax] = s
            diff = F(F(F(d[0] * d[0]) + F(d[1] * d[1])) + F(d[2] * d[2]))
            curv[i] = diff
            p, q = c[i, :3], c[i + 1, :3]
            dis = F(F(F(p[0] * p[0]) + F(p[1] * p[1])) + F(p[2] * p[2]))
            if float(diff) > 0.1:
                d1 = np.sqrt(dis)
                d2 = np.sqrt(F(F(F(q[0] * q[0]) + F(q[1] * q[1])) + F(q[2] * q[2])))
                if d1 > d2:
                    e = [F(q[a] - F(F(p[a] * d2) / d1)) for a in range(3)]
                    occl[i] = float(F(np.sqrt(F(F(F(e[0] * e[0]) + F(e[1] * e[1])) + F(e[2] * e[2]))) / d2)) < 0.1
            g = [F(p[a] - c[i - 1, a]) for a in range(3)]
            diff2 = F(F(F(g[0] * g[0]) + F(g[1] * g[1])) + F(g[2] * g[2]))
            beam[i] = float(diff) > 0.0002 * float(dis) and float(diff2) > 0.0002 * float(dis)
        gx = np.diff(c[:, :3], axis=0)
        cut = np.zeros(N + 1, bool)
        if N > 1:
            cut[1:N] = ((gx[:, 0] * gx[:, 0] + gx[:, 1] * gx[:, 1]) + gx[:, 2] * gx[:, 2]).astype(np.float64) > 0.05
    picked = np.zeros(N + 1, bool)
    for k in range(5, N - 5):
        picked[k] = beam[k] or occl[k:min(k + 5, N - 6) + 1].any()
    picked_before = picked[:N].astype(np.int32)
    label = np.zeros(N, np.int32)

    def mark(ind, cap):
        picked[ind] = True
        for l in range(1, cap + 1):
            if ind + l > N - 1 or cut[ind + l]:
                break
            picked[ind + l] = True
        for l in range(1, cap + 1):
            if ind - l < 0 or cut[ind - l + 1]:
                break
            picked[ind - l] = True

    sharp, less_sharp, flat, less_flat = [], [], [], []
    for r in range(scan_line):
        lf = []
        for j in range(6):
            sp = int((start[r] * (6 - j) + end[r] * j) / 6)        # C division truncates toward zero
            ep = int((start[r] * (5 - j) + end[r] * (j + 1)) / 6) - 1
            if ep < sp:
                continue
            idx = sp + np.argsort(curv[sp:ep + 1], kind="stable")
            n = 0
            for ind in idx[::-1]:
                if not picked[ind] and curv[ind] > F(0.5):
                    n += 1
                    if n > 200:
                        break
                    label[ind] = 2 if n <= 20 else 1
                    (sharp.append(c[ind]) if n <= 20 else None)
                    less_sharp.append(c[ind])
                    mark(ind, 500)
            n = 0
            for ind in idx:
                if not picked[ind] and curv[ind] < F(0.05):
                    label[ind] = -1
                    flat.append(c[ind])
                    n += 1
                    if n >= 5:
                        break
                    mark(ind, 5)
            lf += [c[k] for k in range(sp, ep + 1) if label[k] <= 0]
        if lf:
            less_flat.append(voxel_grid(np.array(lf, np.float32), F(F(plane_resolution) / F(2))))
    as4 = lambda a: np.array(a, np.float32).reshape(-1, 4)
    return ({"full": c, "sharp": as4(sharp), "less_sharp": as4(less_sharp), "flat": as4(flat),
             "less_flat": np.vstack(less_flat) if less_flat else np.zeros((0, 4), np.float32)},
            (np.array(ring, np.int32), curv, picked_before, label))
