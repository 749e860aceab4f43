"""The keyframe oracle (oracle/orc_keyframe.hpp through tests/cpp/keyframe_oracle.cpp) for the tests, NumPy restatements of the loop search's
gates, the keyframe's ROI range and its direction count images, and fp64 references of the blur and the normalised correlation."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PIX = 3600
_LIB = None


def lib():
    """Compiles the oracle shim once per process into a temporary directory, removed at exit."""
    global _LIB
    if _LIB is None:
        d = tempfile.mkdtemp(prefix="keyframe_oracle_")
        atexit.register(shutil.rmtree, d, True)
        out = os.path.join(d, "libkforacle.so")
        r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-w", "-shared", "-fPIC", "-o", out,
                            os.path.join(ROOT, "tests", "cpp", "keyframe_oracle.cpp")], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        L = C.CDLL(out)
        vp = C.c_void_p
        L.kfo_create.restype = vp
        L.kfo_create.argtypes = [C.c_float, C.c_int, C.c_int]
        for n in ("kfo_release", "kfo_new_keyframe", "kfo_cell_count"):
            getattr(L, n).argtypes = [vp]
        L.kfo_append.argtypes = [vp, vp, C.c_int, vp, C.c_int]
        L.kfo_analyze.argtypes = [vp, C.c_int]
        L.kfo_info.argtypes = [vp, C.c_int, vp, vp]
        L.kfo_cells.argtypes = [vp, C.c_int, vp, vp, vp, vp]
        L.kfo_images.argtypes = [vp, C.c_int, vp]
        L.kfo_cloud.argtypes = [vp, C.c_int, C.c_int, vp, C.c_int]
        L.kfo_cell_type.argtypes = [vp, C.c_int, vp, C.c_float, C.c_int, vp, vp, vp]
        L.kfo_eig3.argtypes = [vp, vp, vp]
        L.kfo_blur.argtypes = [vp, vp]
        L.kfo_similarity.argtypes = [vp, vp]
        L.kfo_similarity.restype = C.c_float
        L.kfo_gaussian_kernel.argtypes = [vp]
        L.kfo_search.argtypes = [vp, vp, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp]
        L.kfo_gates.argtypes = [vp, vp, vp, vp, vp, C.c_int, vp, vp, vp, vp]
        _LIB = L
    return _LIB


def _p(a):
    return C.c_void_p(a.ctypes.data)


class OracleMap:
    """The reference's full-resolution cell map with its keyframes (append_cloud + add_cells, Maps_keyframe::analyze)."""

    def __init__(self, resolution=1.0, revisit_threshold=2147483647, incremental=False):
        self.L = lib()
        self.h = C.c_void_p(self.L.kfo_create(resolution, revisit_threshold, int(incremental)))

    def __del__(self):
        if getattr(self, "h", None):
            self.L.kfo_release(self.h)
            self.h = None

    def new_keyframe(self):
        return self.L.kfo_new_keyframe(self.h)

    def append(self, pts, open_kfs):
        p = np.zeros((len(pts), 4), np.float32)
        p[:, :3] = np.asarray(pts, np.float32)[:, :3]
        o = np.ascontiguousarray(open_kfs, np.int32)
        self.L.kfo_append(self.h, _p(p), p.shape[0], _p(o), o.shape[0])

    def cell_count(self):
        return self.L.kfo_cell_count(self.h)

    def analyze(self, k):
        self.L.kfo_analyze(self.h, k)

    def info(self, k):
        fo, io = np.zeros(6, np.float32), np.zeros(4, np.int32)
        self.L.kfo_info(self.h, k, _p(fo), _p(io))
        return dict(center=fo[:3].copy(), roi_range=fo[3], ratio_line=fo[4], ratio_plane=fo[5], cells=int(io[0]), line_cells=int(io[1]),
                    plane_cells=int(io[2]), accumulate_frames=int(io[3]))

    def cells(self, k):
        n = self.info(k)["cells"]
        keys, inc, typ, vec = np.zeros(n, np.uint64), np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros((n, 3), np.float32)
        self.L.kfo_cells(self.h, k, _p(keys), _p(inc), _p(typ), _p(vec))
        return keys, inc, typ, vec

    def images(self, k):
        out = np.zeros((4, 60, 60), np.float32)
        self.L.kfo_images(self.h, k, _p(out))
        return out

    def cloud(self, k, which):
        n = self.L.kfo_cloud(self.h, k, which, None, 0)
        out = np.zeros((max(n, 1), 4), np.float32)
        self.L.kfo_cloud(self.h, k, which, _p(out), n)
        return out[:n]


def cell_type(pts, center, res=0.5, incremental=False):
    """(type, vec, mean, cov) of one constructed cell (Points_cloud_cell::append_pt over pts, then determine_feature)."""
    p = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    c = np.ascontiguousarray(center, np.float32)
    vec, mean, cov = np.zeros(3, np.float32), np.zeros(3, np.float32), np.zeros(9, np.float32)
    t = lib().kfo_cell_type(_p(p), p.shape[0], _p(c), res, int(incremental), _p(vec), _p(mean), _p(cov))
    return t, vec, mean, cov.reshape(3, 3)


def eig3(A):
    A = np.ascontiguousarray(A, np.float64).reshape(9)
    w, V = np.zeros(3), np.zeros(9)
    lib().kfo_eig3(_p(A), _p(w), _p(V))
    return w, V.reshape(3, 3)


def blur(img):
    a = np.ascontiguousarray(img, np.float32)
    out = np.zeros((60, 60), np.float32)
    lib().kfo_blur(_p(a), _p(out))
    return out


def similarity(a, b):
    a = np.ascontiguousarray(a, np.float32)
    b = np.ascontiguousarray(b, np.float32)
    return float(lib().kfo_similarity(_p(a), _p(b)))


def gaussian_kernel():
    k = np.zeros(9, np.float32)
    lib().kfo_gaussian_kernel(_p(k))
    return k


DEFAULT_CFG = dict(minimum_keyframe_differen=200, avail_ratio_plane=0.05, avail_ratio_line=0.03, maximum_roi_difference=5.0,
                   minimum_similarity_linear=0.65, minimum_similarity_planar=0.94, plane_with_line=0.92)


def _cfg_arrays(cfg):
    icfg = np.array([cfg["minimum_keyframe_differen"]], np.int32)
    fcfg = np.array([cfg[k] for k in ("avail_ratio_plane", "avail_ratio_line", "maximum_roi_difference", "minimum_similarity_linear",
                                      "minimum_similarity_planar")], np.float32)
    return icfg, fcfg, np.array([cfg["plane_with_line"]], np.float64)


def oracle_gates(cells, roi, ratio_plane, ratio_line, sims, newest, cfg=DEFAULT_CFG):
    icfg, fcfg, dcfg = _cfg_arrays(cfg)
    a = [np.ascontiguousarray(x, t) for x, t in ((cells, np.int64), (roi, np.float32), (ratio_plane, np.float32), (ratio_line, np.float32),
                                                 (sims, np.float32))]
    cand = np.zeros(max(newest, 1), np.int32)
    n = lib().kfo_gates(*[_p(x) for x in a], newest, _p(icfg), _p(fcfg), _p(dcfg), _p(cand))
    return cand[:n].tolist()


def oracle_search(cells, roi, ratio_plane, ratio_line, imgs, newest, cfg=DEFAULT_CFG):
    """imgs: [n, 2, 60, 60] (plane, line).  Returns (sims [newest, 2], candidates)."""
    icfg, fcfg, dcfg = _cfg_arrays(cfg)
    a = [np.ascontiguousarray(x, t) for x, t in ((cells, np.int64), (roi, np.float32), (ratio_plane, np.float32), (ratio_line, np.float32),
                                                 (imgs, np.float32))]
    sims, cand = np.zeros((max(newest, 1), 2), np.float32), np.zeros(max(newest, 1), np.int32)
    n = lib().kfo_search(*[_p(x) for x in a], newest, _p(icfg), _p(fcfg), _p(dcfg), _p(sims), _p(cand))
    return sims[:newest], cand[:n].tolist()


def numpy_gates(cells, roi, ratio_plane, ratio_line, sims, newest, cfg=DEFAULT_CFG):
    """laser_mapping.hpp:994-1033 in NumPy scalars: size_t arithmetic as uint64, float values as float32, the double literal 0.92 as float64."""
    out = []
    n_kf = np.uint64(newest + 1)
    f32 = np.float32
    for his in range(newest):
        if n_kf - np.uint64(his) < np.uint64(cfg["minimum_keyframe_differen"]):
            continue
        if f32(ratio_plane[his]) < f32(cfg["avail_ratio_plane"]) and f32(ratio_line[his]) < f32(cfg["avail_ratio_line"]):
            continue
        if np.float64(abs(f32(roi[his]) - f32(roi[newest]))) > np.float64(f32(cfg["maximum_roi_difference"])):
            continue
        sp, sl = f32(sims[his][0]), f32(sims[his][1])
        if not ((sl > f32(cfg["minimum_similarity_linear"]) and np.float64(sp) > np.float64(cfg["plane_with_line"]))
                or sp > f32(cfg["minimum_similarity_planar"])):
            continue
        a, b = np.uint64(cells[newest]), np.uint64(cells[his])
        if a + b == 0:
            continue
        with np.errstate(over="ignore"):
            q = (a - b) // (a + b)
        if np.float64(q) * 0.1:
            continue
        out.append(his)
    return out


def numpy_roi_range(centers):
    """get_ratio_range_of_cell(ratio 0.9): centre = float sum of the cell centres times (float)(1.0 / n); distinct float distances (Eigen's norm
    order), element ceil((u - 1) * 0.9f)."""
    c = np.zeros(3, np.float32)
    for p in np.asarray(centers, np.float32):
        c = (c + p).astype(np.float32)
    c = (c * np.float32(1.0 / float(np.float32(len(centers))))).astype(np.float32)
    d = np.asarray(centers, np.float32) - c
    n = np.sqrt((d[:, 0] * d[:, 0] + (d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])).astype(np.float32)).astype(np.float32)
    u = np.unique(n)
    return c, u[int(np.ceil(np.float32(len(u) - 1) * np.float32(0.9)))]


def numpy_images(types, vecs):
    """The direction count images of analyze (:1487-1494) from the cell types and vectors: basis = eigenvectors of I + sum v v^T over plane cells
    (fp64), reversed, column 2 = column 0 x column 1 (float); each vector's bin from the float of the double atan2 / asin.  Returns (line counts,
    plane counts, the image frame coordinates [n, 3] of every vector)."""
    types, vecs = np.asarray(types), np.asarray(vecs, np.float32)
    M = np.eye(3)
    for v in vecs[types == 2]:
        M += np.outer(v, v).astype(np.float32).astype(np.float64)
    _, V = eig3(M)
    R = np.c_[V[:, 2], V[:, 1]].astype(np.float32)
    r0, r1 = R[:, 0], R[:, 1]
    R = np.c_[R, np.array([r0[1] * r1[2] - r0[2] * r1[1], r0[2] * r1[0] - r0[0] * r1[2], r0[0] * r1[1] - r0[1] * r1[0]], np.float32)]
    imgs = np.zeros((2, 60, 60), np.float32)
    frame = np.zeros((len(vecs), 3), np.float32)
    for r, (t, v) in enumerate(zip(types, vecs)):
        if t not in (1, 2):
            continue
        a = np.array([R[0, c] * v[0] + (R[1, c] * v[1] + R[2, c] * v[2]) for c in range(3)], np.float32)   # Eigen's dot order, in float
        frame[r] = a
        if a[0] < 0:
            a = -a
        phi = np.float64(np.float32(np.arctan2(np.float64(a[1]), np.float64(a[0])))) + np.pi / 2
        th = np.float64(np.float32(np.arcsin(np.float64(a[2])))) + np.pi / 2
        pi, ti = (min(max(int(np.floor(x / (np.pi / 60))), 0), 59) for x in (phi, th))
        imgs[0 if t == 1 else 1, pi, ti] += 1
    return imgs[0], imgs[1], frame


def fp64_gaussian_kernel():
    t = np.exp(-((np.arange(9) - 4.0) ** 2) / (2.0 * 16.0))
    return t / t.sum()


def fp64_blur(img):
    """apply_guassian_blur(img, 4, 4) in fp64: the circular 9 x 9 Gaussian (sigma 4) of the 60 x 60 image."""
    g = fp64_gaussian_kernel()
    a = np.asarray(img, np.float64)
    out = np.zeros((60, 60))
    for s in range(9):
        for t in range(9):
            out += g[s] * g[t] * np.roll(a, (4 - s, 4 - t), axis=(0, 1))
    return out


def fp64_similarity(a, b):
    """CCORR_NORMED of the template a over b wrap-padded by 30, in fp64, max over the 61 x 61 positions (0 at a zero norm)."""
    T = np.asarray(a, np.float64)
    P = np.pad(np.asarray(b, np.float64), 30, mode="wrap")
    W = np.lib.stride_tricks.sliding_window_view(P, (60, 60))
    num = np.einsum("yxrc,rc->yx", W, T)
    den = np.einsum("yxrc,yxrc->yx", W, W)
    t = np.sqrt(den * (T * T).sum())
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(t > 0, num / np.where(t > 0, t, 1.0), 0.0)
    return float(r.max())
