"""NumPy restatement of relocalization (ll_reloc_index_build, ll_reloc_scores, the peaks and candidates of ll_relocalize; include/loamlivox_b200.h,
DESIGN.md §4.3), bit for bit: the cells in fp64, the score transform in fp64 with Eigen's association (exact_math.cuh qrot_d), rounded to fp32.
`scores` loops over hypotheses; `scores_vec` computes the same over chunks of translations x score points, fast enough for the shipped search sizes."""
import numpy as np


def finite_bbox(clouds):
    """(lo, hi) float32 [3] of the finite points of the clouds (what the map's d_bbox holds), or None."""
    pts = np.concatenate([np.asarray(c, np.float32)[:, :3] for c in clouds], axis=0)
    pts = pts[np.all(np.isfinite(pts), axis=1)]
    if pts.shape[0] == 0:
        return None
    return pts.min(axis=0), pts.max(axis=0)


def dims_of(lo, hi, res, dilate):
    res = float(np.float32(res))
    return np.array([int(np.floor((float(hi[a]) - float(lo[a])) / res)) + 1 + 2 * dilate for a in range(3)], np.int64)


def cells(p, lo, res, dilate, dims):
    """[n, 3] int64 cells of float32 points p and a bool mask of those inside the grid (fp64, compared as doubles)."""
    p = np.asarray(p, np.float32)[:, :3].astype(np.float64)
    with np.errstate(invalid="ignore"):
        d = np.floor((p - np.asarray(lo, np.float32).astype(np.float64)) / float(np.float32(res))) + float(dilate)
        ok = np.all((d >= 0.0) & (d < dims.astype(np.float64)), axis=1)
    c = np.zeros(d.shape, np.int64)
    c[ok] = d[ok].astype(np.int64)
    return c, ok


def occupancy(clouds, res, dilate):
    """(dims, lo, occ [dims2, dims1, dims0] bool) before dilation."""
    lo, hi = finite_bbox(clouds)
    dims = dims_of(lo, hi, res, dilate)
    occ = np.zeros((dims[2], dims[1], dims[0]), bool)
    for c in clouds:
        c = np.asarray(c, np.float32)
        c = c[np.all(np.isfinite(c[:, :3]), axis=1)]
        ci, ok = cells(c, lo, res, dilate, dims)
        ci = ci[ok]
        occ[ci[:, 2], ci[:, 1], ci[:, 0]] = True
    return dims, lo, occ


def dilate_separable(occ, r):
    """Chebyshev dilation of radius r by three separable passes (clipped at the border)."""
    out = occ.copy()
    for ax in range(3):
        src, out = out, np.zeros_like(out)
        n = src.shape[ax]
        for k in range(-r, r + 1):
            a, b = max(0, -k), min(n, n - k)   # out[i] |= src[i + k] for i in [a, b)
            if a >= b:
                continue
            sl_o = [slice(None)] * 3
            sl_s = [slice(None)] * 3
            sl_o[ax] = slice(a, b)
            sl_s[ax] = slice(a + k, b + k)
            out[tuple(sl_o)] |= src[tuple(sl_s)]
    return out


def pack_words(grid):
    """[dims2, dims1, dims0] bool -> uint32 words, voxel v = x + dims0 (y + dims1 z) in bit v & 31 of word v >> 5."""
    bits = grid.reshape(-1)
    n_words = (bits.shape[0] + 31) // 32
    pad = np.zeros(n_words * 32, bool)
    pad[:bits.shape[0]] = bits
    return np.packbits(pad.reshape(-1, 32)[:, ::-1], axis=1).view(">u4").astype(np.uint32).reshape(-1)


def index(clouds, res, dilate):
    """(dims int64 [3], lo float32 [3], dilated grid bool [dims2, dims1, dims0], words uint32)."""
    dims, lo, occ = occupancy(clouds, res, dilate)
    g = dilate_separable(occ, dilate) if dilate > 0 else occ
    return dims, lo, g, pack_words(g)


def qrot(q, p):
    """exact_math.cuh qrot_d over [n, 3] fp64 points: uv = 2 (u x v); v + w uv + u x uv, in that association."""
    w, ux, uy, uz = (float(v) for v in q)
    vx, vy, vz = p[:, 0], p[:, 1], p[:, 2]
    cx = uy * vz - uz * vy
    cy = uz * vx - ux * vz
    cz = ux * vy - uy * vx
    cx = cx + cx
    cy = cy + cy
    cz = cz + cz
    dx = uy * cz - uz * cy
    dy = uz * cx - ux * cz
    dz = ux * cy - uy * cx
    return np.stack([(vx + cx * w) + dx, (vy + cy * w) + dy, (vz + cz * w) + dz], axis=1)


def lattice(t0, step, nt):
    """[nt2 * nt1 * nt0, 3] translations, x fastest: t = t0 + i * step (fp64)."""
    i, j, k = np.meshgrid(np.arange(nt[0]), np.arange(nt[1]), np.arange(nt[2]), indexing="ij")
    i, j, k = i.transpose(2, 1, 0).reshape(-1), j.transpose(2, 1, 0).reshape(-1), k.transpose(2, 1, 0).reshape(-1)
    return np.stack([t0[0] + i.astype(np.float64) * step[0], t0[1] + j.astype(np.float64) * step[1], t0[2] + k.astype(np.float64) * step[2]], axis=1)


def scores(grid, dims, lo, res, dilate, pts, rot, t0, step, nt):
    """int32 score of every hypothesis h = l + n_lat * r."""
    p = np.asarray(pts, np.float32)[:, :3]
    fin = np.all(np.isfinite(p), axis=1)
    p = p[fin].astype(np.float64)
    T = lattice(t0, step, nt)
    flat = grid.reshape(-1)
    out = np.zeros(len(rot) * T.shape[0], np.int32)
    for r, q in enumerate(rot):
        rp = qrot(q, p)
        for l in range(T.shape[0]):
            pw = (rp + T[l]).astype(np.float32)
            c, ok = cells(pw, lo, res, dilate, dims)
            v = c[ok, 0] + dims[0] * (c[ok, 1] + dims[1] * c[ok, 2])
            out[r * T.shape[0] + l] = int(np.count_nonzero(flat[v]))
    return out


CHUNK_ELEMS = 1 << 20   # lattice points x score points per chunk of the vectorised scorers: each [chunk, n, 3] fp64 temporary is 24 MB


def finite_points(pts):
    """The score points with three finite coordinates, fp64 [n, 3] (the kernels rotate a non-finite point to NaN, which never scores)."""
    p = np.asarray(pts, np.float32).reshape(-1, 4)[:, :3]
    return p[np.all(np.isfinite(p), axis=1)].astype(np.float64)


def flat_cells(pw, lo, res, pad, dims):
    """`cells` over fp32 points [..., 3] of any shape, as flat voxels v = x + dims0 (y + dims1 z) ([...] int64, 0 outside) and the mask of those
    inside the grid."""
    dims = np.asarray(dims, np.int64)
    with np.errstate(invalid="ignore", over="ignore"):
        d = np.floor((pw.astype(np.float64) - np.asarray(lo, np.float32).astype(np.float64)) / float(np.float32(res))) + float(pad)
        ok = np.all((d >= 0.0) & (d < dims.astype(np.float64)), axis=-1)
    c = np.where(ok[..., None], d, 0.0).astype(np.int64)
    return c[..., 0] + dims[0] * (c[..., 1] + dims[1] * c[..., 2]), ok


def lattice_sums(rp, T, value, lo, res, pad, dims, chunk=None):
    """[n_lat] int64: for every translation T[l] (fp64), the sum of value[v] over the rotated points rp [n, 3] (fp64) whose p_w = fp32(rp + T[l])
    lands in voxel v of the grid.  `chunk` translations at a time (default CHUNK_ELEMS / n): the per-hypothesis loop of `scores`, vectorised with
    the same arithmetic element for element."""
    out = np.zeros(T.shape[0], np.int64)
    if rp.shape[0] == 0 or T.shape[0] == 0:
        return out
    c = int(chunk) if chunk else max(1, CHUNK_ELEMS // rp.shape[0])
    for l0 in range(0, T.shape[0], c):
        v, ok = flat_cells((rp[None, :, :] + T[l0:l0 + c, None, :]).astype(np.float32), lo, res, pad, dims)
        out[l0:l0 + c] = np.where(ok, value[v], 0).sum(axis=1)
    return out


def scores_vec(grid, dims, lo, res, dilate, pts, rot, t0, step, nt, chunk=None):
    """`scores`, vectorised over chunks of translations x score points."""
    p = finite_points(pts)
    T = lattice(t0, step, nt)
    flat = grid.reshape(-1).astype(np.int64)
    out = [lattice_sums(qrot(q, p), T, flat, lo, res, dilate, dims, chunk) for q in rot]
    return np.concatenate(out).astype(np.int32) if out else np.zeros(0, np.int32)


def relocalize(grid, dims, lo, res, dilate, pts, rot, t0, step, nt, K, cyclic=True, chunk=None):
    """One ll_relocalize call up to the refinement: coarse scores -> peaks -> the first K.  {"scores", "n_peaks", "candidates": [{hypothesis,
    score, q, t}]}."""
    sc = scores_vec(grid, dims, lo, res, dilate, pts, rot, t0, step, nt, chunk)
    hs, ss = peaks(sc, len(rot), nt, cyclic)
    cands = []
    for h, s in zip(hs[:K], ss[:K]):
        q, t = candidate_pose(h, rot, t0, step, nt)
        cands.append({"hypothesis": int(h), "score": int(s), "q": q, "t": t})
    return {"scores": sc, "n_peaks": int(hs.shape[0]), "candidates": cands}


def scores_loop(grid, dims, lo, res, dilate, pts, rot, t0, step, nt):
    """The same as a plain per-point loop (the test's second restatement)."""
    flat = grid.reshape(-1)
    T = lattice(t0, step, nt)
    out = np.zeros(len(rot) * T.shape[0], np.int32)
    res64, lo64 = float(np.float32(res)), [float(v) for v in np.asarray(lo, np.float32)]
    for r, q in enumerate(rot):
        for l in range(T.shape[0]):
            n = 0
            for p in np.asarray(pts, np.float32):
                if not (np.isfinite(p[0]) and np.isfinite(p[1]) and np.isfinite(p[2])):
                    continue
                rp = qrot(q, p[None, :3].astype(np.float64))[0]
                c = []
                for a in range(3):
                    x = float(np.float32(rp[a] + T[l, a]))
                    d = np.floor((x - lo64[a]) / res64) + dilate
                    if not (0.0 <= d < dims[a]):
                        break
                    c.append(int(d))
                else:
                    n += int(flat[c[0] + dims[0] * (c[1] + dims[1] * c[2])])
            out[r * T.shape[0] + l] = n
    return out


def peaks(sc, n_rot, nt, cyclic):
    """The peaks in (score descending, index ascending) order: h with score >= 1 that comes first among its lattice Chebyshev-1 neighbours (clipped)
    at rotations r - 1, r, r + 1 (wrapped when cyclic and n_rot >= 3).  Vectorised over shifted copies of the score field."""
    nt0, nt1, nt2 = nt
    S = np.asarray(sc, np.int64).reshape(n_rot, nt2, nt1, nt0)
    H = np.arange(S.size, dtype=np.int64).reshape(S.shape)
    is_peak = S >= 1
    wrap = cyclic and n_rot >= 3
    for dr in (-1, 0, 1):
        for dk in (-1, 0, 1):
            for dj in (-1, 0, 1):
                for di in (-1, 0, 1):
                    if dr == dk == dj == di == 0:
                        continue
                    S2 = np.full(S.shape, -1, np.int64)
                    H2 = np.full(S.shape, -1, np.int64)
                    src = [slice(None)] * 4
                    dst = [slice(None)] * 4
                    ok = True
                    for ax, d, n in ((0, dr, n_rot), (1, dk, nt2), (2, dj, nt1), (3, di, nt0)):
                        if ax == 0 and wrap:
                            continue
                        if d >= n or -d >= n:
                            ok = False
                            break
                        dst[ax] = slice(max(0, -d), n - max(0, d))
                        src[ax] = slice(max(0, d), n - max(0, -d))
                    if not ok:
                        continue
                    Ssrc, Hsrc = (np.roll(S, -dr, axis=0), np.roll(H, -dr, axis=0)) if wrap else (S, H)
                    S2[tuple(dst)] = Ssrc[tuple(src)]
                    H2[tuple(dst)] = Hsrc[tuple(src)]
                    beaten = (S2 > S) | ((S2 == S) & (H2 >= 0) & (H2 < H))
                    is_peak &= ~beaten
    h = H[is_peak]
    s = S[is_peak]
    order = np.lexsort((h, -s))
    return h[order], s[order]


def peaks_brute(sc, n_rot, nt, cyclic):
    """The same by a plain neighbourhood loop."""
    nt0, nt1, nt2 = nt
    n_lat = nt0 * nt1 * nt2
    out = []
    for h in range(len(sc)):
        s = int(sc[h])
        if s < 1:
            continue
        r, l = divmod(h, n_lat)
        i, j, k = l % nt0, (l // nt0) % nt1, l // (nt0 * nt1)
        rs = set()
        for dr in (-1, 0, 1):
            rr = r + dr
            if cyclic and n_rot >= 3:
                rr %= n_rot
            elif not 0 <= rr < n_rot:
                continue
            rs.add(rr)
        best = True
        for rr in rs:
            for kk in range(max(0, k - 1), min(nt2, k + 2)):
                for jj in range(max(0, j - 1), min(nt1, j + 2)):
                    for ii in range(max(0, i - 1), min(nt0, i + 2)):
                        h2 = ii + nt0 * (jj + nt1 * kk) + n_lat * rr
                        if h2 != h and (sc[h2] > s or (sc[h2] == s and h2 < h)):
                            best = False
        if best:
            out.append((h, s))
    out.sort(key=lambda e: (-e[1], e[0]))
    return np.array([e[0] for e in out], np.int64), np.array([e[1] for e in out], np.int64)


def candidate_pose(h, rot, t0, step, nt):
    """(q, t) of hypothesis h."""
    n_lat = nt[0] * nt[1] * nt[2]
    r, l = divmod(int(h), n_lat)
    i, j, k = l % nt[0], (l // nt[0]) % nt[1], l // (nt[0] * nt[1])
    return np.asarray(rot[r], np.float64), np.array([t0[0] + float(i) * step[0], t0[1] + float(j) * step[1], t0[2] + float(k) * step[2]])
