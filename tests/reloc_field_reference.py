"""NumPy restatement of relocalization by class-aware distance fields (ll_reloc_field_build, ll_reloc_field_scores, the fine groups and picks of
ll_relocalize_field; include/loamlivox_b200.h, DESIGN.md §4.3.1), bit for bit.  The grid, the cells, the lattice, the score transform and the
peaks are those of the occupancy relocalization (tests/reloc_reference.py).  `field_scores` loops over hypotheses; `field_scores_vec` and the
one-call pipeline `relocalize_field` are fast enough for the shipped search sizes."""
import numpy as np

from reloc_reference import candidate_pose, cells, dims_of, finite_bbox, finite_points, lattice, lattice_sums, peaks, qrot


def class_occupancy(clouds, res, T):
    """(dims, lo, [occ per cloud] bool [dims2, dims1, dims0]): one grid anchored at the finite bounding box of all clouds, padded by T."""
    lo, hi = finite_bbox(clouds)
    dims = dims_of(lo, hi, res, T)
    occs = []
    for c in clouds:
        occ = np.zeros((dims[2], dims[1], dims[0]), bool)
        c = np.asarray(c, np.float32)
        c = c[np.all(np.isfinite(c[:, :3]), axis=1)] if c.shape[0] else c.reshape(0, 4)
        ci, ok = cells(c, lo, res, T, dims)
        ci = ci[ok]
        occ[ci[:, 2], ci[:, 1], ci[:, 0]] = True
        occs.append(occ)
    return dims, lo, occs


def edt_separable(occ, T):
    """The truncated squared distance transform by the three passes of reloc_edt_kernel (x, then y, then z; absent past the border), uint8."""
    T2 = T * T
    g = None   # before the first pass: the occupancy itself
    for ax in (2, 1, 0):   # numpy axes of x, y, z
        n = occ.shape[ax]
        out = np.full(occ.shape, T2, np.int64)
        for k in range(-T, T + 1):
            a, b = max(0, -k), min(n, n - k)   # out[i] = min(out[i], term(i + k)) for i in [a, b)
            if a >= b:
                continue
            so, ss = [slice(None)] * 3, [slice(None)] * 3
            so[ax], ss[ax] = slice(a, b), slice(a + k, b + k)
            term = np.where(occ[tuple(ss)], k * k, T2) if g is None else g[tuple(ss)] + k * k
            out[tuple(so)] = np.minimum(out[tuple(so)], term)
        g = np.minimum(out, T2)
    return g.astype(np.uint8)


def field(clouds, res, T):
    """(dims, lo, [d2 corner, d2 surface] uint8 [dims2, dims1, dims0]) of ll_reloc_field_build over clouds = [corner, surface]."""
    dims, lo, occs = class_occupancy(clouds, res, T)
    return dims, lo, [edt_separable(o, T) for o in occs]


def field_scores(d2, dims, lo, res, T, pts, rot, t0, step, nt):
    """int32 field score of every hypothesis h = l + n_lat * r (pts = [corner, surface] score points)."""
    T2 = T * T
    Tl = lattice(t0, step, nt)
    out = np.zeros(len(rot) * Tl.shape[0], np.int64)
    for cls in range(2):
        p = np.asarray(pts[cls], np.float32).reshape(-1, 4)[:, :3]
        p = p[np.all(np.isfinite(p), axis=1)].astype(np.float64)
        flat = d2[cls].reshape(-1).astype(np.int64)
        for r, q in enumerate(rot):
            rp = qrot(q, p)
            for l in range(Tl.shape[0]):
                c, ok = cells((rp + Tl[l]).astype(np.float32), lo, res, T, dims)
                v = c[ok, 0] + dims[0] * (c[ok, 1] + dims[1] * c[ok, 2])
                out[r * Tl.shape[0] + l] += int(np.sum(T2 - flat[v]))
    return out.astype(np.int32)


def field_scores_vec(d2, dims, lo, res, T, pts, rot, t0, step, nt, chunk=None):
    """`field_scores`, vectorised over chunks of translations x score points (reloc_reference.lattice_sums)."""
    Tl = lattice(t0, step, nt)
    out = np.zeros(len(rot) * Tl.shape[0], np.int64)
    for cls in range(2):
        p = finite_points(pts[cls])
        value = T * T - d2[cls].reshape(-1).astype(np.int64)
        for r, q in enumerate(rot):
            out[r * Tl.shape[0]:(r + 1) * Tl.shape[0]] += lattice_sums(qrot(q, p), Tl, value, lo, res, T, dims, chunk)
    return out.astype(np.int32)


def relocalize_field(d2, dims, lo, res, T, pts, rot, t0, step, nt, K, dq, fstep, fnt, cyclic=True, chunk=None):
    """One ll_relocalize_field call up to the refinement: coarse scores -> peaks -> the first K -> their fine groups -> each group's pick -> the
    fine poses.  {"scores", "n_peaks", "fine": [each group's scores], "candidates": [{hypothesis, score, q, t, fine_index, fine_score, fine_q,
    fine_t}]}."""
    sc = field_scores_vec(d2, dims, lo, res, T, pts, rot, t0, step, nt, chunk)
    hs, ss = peaks(sc, len(rot), nt, cyclic)
    fine, cands = [], []
    for h, s in zip(hs[:K], ss[:K]):
        q, t = candidate_pose(h, rot, t0, step, nt)
        rf, o = fine_group(q, t, dq, fstep, fnt)
        fs = field_scores_vec(d2, dims, lo, res, T, pts, rf, o, fstep, fnt, chunk)
        i, s_f = pick(fs)
        fq, ft = fine_pose(rf, o, fstep, fnt, i)
        fine.append(fs)
        cands.append({"hypothesis": int(h), "score": int(s), "q": q, "t": t, "fine_index": i, "fine_score": s_f, "fine_q": fq, "fine_t": ft})
    return {"scores": sc, "n_peaks": int(hs.shape[0]), "fine": fine, "candidates": cands}


def verify_scores(d2, dims, lo, res, T, pts, poses):
    """The field score at each (q, t) of `poses`: ll_relocalize_field's verify step at the refined poses."""
    return [int(field_scores_vec(d2, dims, lo, res, T, pts, np.asarray(q, np.float64)[None], tuple(t), (0.0, 0.0, 0.0), (1, 1, 1))[0]) for q, t in poses]


def field_scores_loop(d2, dims, lo, res, T, pts, rot, t0, step, nt):
    """The same as a plain per-point loop."""
    Tl = lattice(t0, step, nt)
    out = np.zeros(len(rot) * Tl.shape[0], np.int64)
    res64, lo64 = float(np.float32(res)), [float(v) for v in np.asarray(lo, np.float32)]
    for r, q in enumerate(rot):
        for l in range(Tl.shape[0]):
            n = 0
            for cls in range(2):
                flat = d2[cls].reshape(-1)
                for p in np.asarray(pts[cls], np.float32).reshape(-1, 4):
                    if not (np.isfinite(p[0]) and np.isfinite(p[1]) and np.isfinite(p[2])):
                        continue
                    rp = qrot(q, p[None, :3].astype(np.float64))[0]
                    c = []
                    for a in range(3):
                        d = np.floor((float(np.float32(rp[a] + Tl[l, a])) - lo64[a]) / res64) + T
                        if not (0.0 <= d < dims[a]):
                            break
                        c.append(int(d))
                    else:
                        n += T * T - int(flat[c[0] + dims[0] * (c[1] + dims[1] * c[2])])
            out[r * Tl.shape[0] + l] = n
    return out.astype(np.int32)


def quat_mul(a, b):
    """The Hamilton product a (x) b in fp64, each component summed left to right (ll_relocalize_field's fine rotations)."""
    w1, x1, y1, z1 = (float(v) for v in a)
    w2, x2, y2, z2 = (float(v) for v in b)
    return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])


def fine_group(q, t, dq, step, nt):
    """(rotations [n_rot, 4], origin [3]) of the fine group around the candidate (q, t): q (x) dq_r and t - ((nt - 1) / 2) * step."""
    return np.array([quat_mul(q, d) for d in dq]), np.array([float(t[a]) - float((int(nt[a]) - 1) // 2) * float(step[a]) for a in range(3)])


def pick(sc):
    """(index, score) of the first hypothesis in (score descending, index ascending)."""
    sc = np.asarray(sc, np.int64)
    i = int(np.argmax(sc))   # argmax returns the first maximum
    return i, int(sc[i])


def fine_pose(rot, origin, step, nt, i):
    """(q, t) of fine index i = l + n_lat * r of a group."""
    n_lat = nt[0] * nt[1] * nt[2]
    r, l = divmod(int(i), n_lat)
    li = (l % nt[0], (l // nt[0]) % nt[1], l // (nt[0] * nt[1]))
    return np.asarray(rot[r], np.float64), np.array([float(origin[a]) + float(li[a]) * float(step[a]) for a in range(3)])
