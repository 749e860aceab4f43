"""Host-side mirror of the reference's C++ interface for the hot path, over the C-ABI (ctypes).

Names, argument meaning and return conventions follow the reference so the parity tests read like its call sites:

  Livox_laser.extract_laser_features / get_features      loam_livox/source/livox_feature_extractor.hpp:722,219
  voxel_grid_filter (pcl::VoxelGrid::filter)             loam_livox/source/laser_mapping.hpp:1367-1373
  Map (update_buff_for_matching's KdTreeFLANN pair)      loam_livox/source/laser_mapping.hpp:533-559
  Point_cloud_registration.find_out_incremental_transfrom / pointcloudAssociateToMap
                                                         loam_livox/source/point_cloud_registration.hpp:163,673
Everything here is plumbing: the arithmetic runs in the CUDA kernels of libloamlivox_b200.so.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import capi
from .capi import LoamLivoxError, _pts


class Context:
    """One CUDA stream + device arenas (the reference creates one Point_cloud_registration per worker thread)."""

    def __init__(self, device: int = 0, **cfg):
        self._lib = capi.lib()
        self.cfg = capi.default_config(**cfg)
        h = C.c_void_p()
        st = self._lib.ll_ctx_create(C.byref(self.cfg), device, C.byref(h))
        if st != capi.LL_OK:
            raise LoamLivoxError(f"ll_ctx_create failed ({st}): a CUDA device (sm_90a) is required, there is no CPU fallback")
        self.h = h
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self._lib.ll_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def check(self, st):
        if st != capi.LL_OK:
            raise LoamLivoxError(f"status {st}: {self._lib.ll_last_error(self.h).decode()}")

    def set_point_layout(self, point_step, offset_x=0, offset_y=4, offset_z=8, offset_intensity=12, intensity_datatype=capi.LL_I_FLOAT32):
        """Record layout of LL_FMT_STRIDED inputs (a sensor_msgs/PointCloud2 payload: what pcl::fromROSMsg resolves by field name)."""
        L = capi.PointLayout(point_step, offset_x, offset_y, offset_z, offset_intensity, intensity_datatype)
        self.check(self._lib.ll_set_point_layout(self.h, C.byref(L)))
        self._layout_step = point_step

    def warmup(self):
        """One toy registration now: first-use costs (module loads, first cooperative launch) are paid here instead of in the first real scan."""
        self.check(self._lib.ll_ctx_warmup(self.h))

    def launches(self) -> int:
        return int(self._lib.ll_launch_count(self.h))

    def sync(self):
        self.check(self._lib.ll_ctx_sync(self.h))

    def stream(self) -> int:
        return int(self._lib.ll_ctx_stream(self.h) or 0)


def format_pose_log(result: capi.RegResult) -> str:
    """One accepted scan in the reference's poses.log format (laser_mapping.hpp:1506-1511)."""
    buf = C.create_string_buffer(1024)
    n = capi.lib().ll_format_pose_log(C.byref(result), buf, 1024)
    if n < 0:
        raise LoamLivoxError("ll_format_pose_log failed")
    return buf.value.decode()


class Livox_laser:
    """Mirror of class Livox_laser (livox_feature_extractor.hpp:77)."""

    def __init__(self, ctx: Context):
        self.ctx = ctx
        self.n = 0
        ctx.check(ctx._lib.ll_extract_reset(ctx.h))   # a new Livox_laser object has no cross-scan history

    def extract_laser_features(self, laserCloudIn, time_stamp: float) -> int:
        """Returns laserCloudScans.size() (number of petals handed back; the caller drops the frame if <= 5)."""
        pts, fmt = _pts(laserCloudIn)
        self.n = pts.shape[0]
        ns = C.c_int(0)
        self.ctx.check(self.ctx._lib.ll_extract(self.ctx.h, pts.ctypes.data, self.n, fmt, capi.LL_HOST, float(time_stamp), C.byref(ns)))
        return ns.value

    def extract_from_pointcloud2(self, data: bytes, n_points: int, time_stamp: float) -> int:
        """Same, from the raw payload of a sensor_msgs/PointCloud2 (layout set with Context.set_point_layout): replaces pcl::fromROSMsg +
        extract_laser_features (laser_feature_extractor.hpp:275,285); the payload is unpacked on the device."""
        buf = np.frombuffer(data, dtype=np.uint8)
        self.n = int(n_points)
        ns = C.c_int(0)
        self.ctx.check(self.ctx._lib.ll_extract(self.ctx.h, buf.ctypes.data, self.n, capi.LL_FMT_STRIDED, capi.LL_HOST, float(time_stamp), C.byref(ns)))
        return ns.value

    def get_features(self, minimum_blur: float = 0.0, maximum_blur: float = 0.3):
        n = self.n
        c = np.empty((n, 4), np.float32)
        s = np.empty((n, 4), np.float32)
        f = np.empty((n, 4), np.float32)
        nc, ns, nf = C.c_size_t(), C.c_size_t(), C.c_size_t()
        self.ctx.check(self.ctx._lib.ll_get_features(self.ctx.h, minimum_blur, maximum_blur, c.ctypes.data, C.byref(nc), s.ctypes.data, C.byref(ns),
                                                     f.ctypes.data, C.byref(nf)))
        return c[:nc.value].copy(), s[:ns.value].copy(), f[:nf.value].copy()

    def piece_bounds(self, pieces: int):
        a = np.empty(pieces, np.float32)
        b = np.empty(pieces, np.float32)
        self.ctx.check(self.ctx._lib.ll_piece_bounds(self.ctx.h, pieces, a.ctypes.data, b.ctypes.data))
        return a, b

    def point_info(self):
        n = self.n
        o = dict(pt_type=np.empty(n, np.int32), pt_label=np.empty(n, np.int32), curvature=np.empty(n, np.float32), view_angle=np.empty(n, np.float32),
                 depth_sq2=np.empty(n, np.float32), time_stamp=np.empty(n, np.float32), polar_dis_sq2=np.empty(n, np.float32), polar_direction=np.empty(n, np.int32))
        self.ctx.check(self.ctx._lib.ll_extract_point_info(self.ctx.h, *[o[k].ctypes.data for k in
                                                                         ("pt_type", "pt_label", "curvature", "view_angle", "depth_sq2", "time_stamp", "polar_dis_sq2", "polar_direction")]))
        return o

    def split_idx(self):
        buf = np.empty(self.n + 1, np.int32)
        m = C.c_int(0)
        self.ctx.check(self.ctx._lib.ll_extract_split_idx(self.ctx.h, buf.ctypes.data, buf.shape[0], C.byref(m)))
        return buf[:m.value].copy()

    def petal_angles(self):
        """Petal angle (scan_id_index) of each segment between consecutive split indices; empty when the scan has fewer than 6 split indices."""
        buf = np.empty(self.n + 1, np.float32)
        m = C.c_int(0)
        self.ctx.check(self.ctx._lib.ll_extract_petal_angles(self.ctx.h, buf.ctypes.data, buf.shape[0], C.byref(m)))
        return buf[:m.value].copy()


def voxel_grid_filter(ctx: Context, cloud, leaf: float):
    """pcl::VoxelGrid<PointXYZI>::setLeafSize(leaf,leaf,leaf) + filter."""
    pts, fmt = _pts(cloud)
    out = np.empty((pts.shape[0], 4), np.float32)
    m = C.c_size_t(0)
    ctx.check(ctx._lib.ll_voxel_downsample(ctx.h, pts.ctypes.data, pts.shape[0], fmt, capi.LL_HOST, leaf, out.ctypes.data, C.byref(m)))
    return out[:m.value].copy()


def voxel_grid_segments(ctx: Context, cloud, seg_end, leaf: float):
    """VoxelGrid over disjoint contiguous segments of one cloud in one device pass (ll_voxel_downsample_segments): segment k is
    cloud[seg_end[k - 1]:seg_end[k]], each filtered as if alone.  Returns the list of per-segment outputs."""
    pts = np.ascontiguousarray(cloud, np.float32).reshape(-1, 4)
    ends = np.ascontiguousarray(seg_end, np.uint64)
    out = np.empty((max(pts.shape[0], 1), 4), np.float32)
    counts = np.zeros(ends.shape[0], np.uint64)
    ctx.check(ctx._lib.ll_voxel_downsample_segments(ctx.h, pts.ctypes.data, pts.shape[0], ends.ctypes.data, ends.shape[0], float(leaf), out.ctypes.data, counts.ctypes.data))
    b = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    return [out[b[k]:b[k + 1]].copy() for k in range(ends.shape[0])]


class Map:
    """The match-map snapshot: two world-frame clouds + their exact-kNN indices (m_kdtree_{corner,surf}_from_map_last)."""

    def __init__(self, ctx: Context, corner, surf, rank: int = 0, world: int = 1, cell_size: float = 2.0):
        self.ctx = ctx
        c, fmt = _pts(corner)
        s, fmt2 = _pts(surf)
        assert fmt == fmt2
        h = C.c_void_p()
        if world > 1:
            st = ctx._lib.ll_map_build_sharded(ctx.h, c.ctypes.data, c.shape[0], s.ctypes.data, s.shape[0], fmt, capi.LL_HOST, rank, world, cell_size,
                                               2.0 ** 0.5, 50.0 ** 0.5, C.byref(h))
        else:
            st = ctx._lib.ll_map_build(ctx.h, c.ctypes.data, c.shape[0], s.ctypes.data, s.shape[0], fmt, capi.LL_HOST, C.byref(h))
        ctx.check(st)
        self.h = h

    def size(self, which):
        return int(self.ctx._lib.ll_map_size(self.h, which))

    def shard_info(self):
        """(ShardInfo, owner table [dims z,y,x] int32) of a sharded snapshot (ll_map_shard_info)."""
        info = capi.ShardInfo()
        self.ctx.check(self.ctx._lib.ll_map_shard_info(self.h, C.byref(info), None, 0))
        owner = np.zeros(int(info.dims[0]) * int(info.dims[1]) * int(info.dims[2]), np.int32)
        self.ctx.check(self.ctx._lib.ll_map_shard_info(self.h, C.byref(info), owner.ctypes.data, owner.shape[0]))
        return info, owner

    def nearestKSearch(self, which: int, queries_world):
        """k = 5 search of either tree; returns (indices [nq,5] int32, squared distances [nq,5] float32)."""
        q = np.ascontiguousarray(queries_world, np.float32)
        idx = np.empty((q.shape[0], 5), np.int32)
        d2 = np.empty((q.shape[0], 5), np.float32)
        self.ctx.check(self.ctx._lib.ll_knn(self.ctx.h, self.h, which, q.ctypes.data, q.shape[0], idx.ctypes.data, d2.ctypes.data))
        return idx, d2

    def release(self):
        if getattr(self, "h", None):
            self.ctx._lib.ll_map_release(self.h)
            self.h = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


class Point_cloud_registration:
    """Mirror of class Point_cloud_registration (point_cloud_registration.hpp:38). Quaternions are (w,x,y,z)."""

    def __init__(self, ctx: Context, **state):
        self.ctx = ctx
        self.state = capi.default_reg_state(**state)
        self.result = capi.RegResult()

    # the members init_pointcloud_registration writes (laser_mapping.hpp:1266-1297) are fields of self.state
    def set_pose(self, q_wxyz, t):
        self.state.q_w_last[:] = list(q_wxyz)
        self.state.t_w_last[:] = list(t)
        self.state.q_w_curr[:] = list(q_wxyz)
        self.state.t_w_curr[:] = list(t)

    def find_out_incremental_transfrom(self, match_map: Map, laserCloudCornerStack, laserCloudSurfStack) -> int:
        c, fmt = _pts(laserCloudCornerStack)
        s, _ = _pts(laserCloudSurfStack)
        self.ctx.check(self.ctx._lib.ll_register(self.ctx.h, match_map.h, c.ctypes.data, c.shape[0], s.ctypes.data, s.shape[0], fmt, capi.LL_HOST,
                                                 C.byref(self.state), C.byref(self.result)))
        r = self.result
        self.m_q_w_curr, self.m_t_w_curr = np.array(r.q_w_curr), np.array(r.t_w_curr)
        self.m_q_w_incre, self.m_t_w_incre = np.array(r.q_w_incre), np.array(r.t_w_incre)
        self.m_inlier_threshold = r.inlier_threshold
        return r.status

    def pointcloudAssociateToMap(self, pc_in, q_wxyz=None, t=None):
        q = np.asarray(self.m_q_w_curr if q_wxyz is None else q_wxyz, np.float64)
        t = np.asarray(self.m_t_w_curr if t is None else t, np.float64)
        p, fmt = _pts(pc_in)
        out = np.empty((p.shape[0], 4), np.float32)
        self.ctx.check(self.ctx._lib.ll_transform(self.ctx.h, q.ctypes.data, t.ctypes.data, p.ctypes.data, p.shape[0], fmt, capi.LL_HOST, out.ctypes.data))
        return out

    # ---- step-by-step parity hooks
    def build_blocks(self, match_map: Map, corner, surf):
        c, fmt = _pts(corner)
        s, _ = _pts(surf)
        M = c.shape[0] + s.shape[0]
        typ = np.zeros(M, np.int32)
        a3 = np.zeros((M, 3))
        v3 = np.zeros((M, 3))
        ca, sa = C.c_int(), C.c_int()
        self.ctx.check(self.ctx._lib.ll_build_blocks(self.ctx.h, match_map.h, c.ctypes.data, c.shape[0], s.ctypes.data, s.shape[0], fmt, capi.LL_HOST, C.byref(self.state),
                                                     typ.ctypes.data, a3.ctypes.data, v3.ctypes.data, C.byref(ca), C.byref(sa)))
        self._hook_slots = M
        return typ, a3, v3, ca.value, sa.value

    def normal_equations(self, x7):
        x = np.ascontiguousarray(x7, np.float64)
        out = np.zeros(28)
        self.ctx.check(self.ctx._lib.ll_normal_equations(self.ctx.h, x.ctypes.data, out.ctypes.data))
        H = np.zeros((6, 6))
        k = 0
        for i in range(6):
            for j in range(i, 6):
                H[i, j] = H[j, i] = out[k]
                k += 1
        return H, out[21:27].copy(), out[27]

    def solve(self, x7, max_iterations):
        x = np.array(x7, np.float64)
        ic, fc, it = C.c_double(), C.c_double(), C.c_int()
        self.ctx.check(self.ctx._lib.ll_solve(self.ctx.h, max_iterations, x.ctypes.data, C.byref(ic), C.byref(fc), C.byref(it)))
        return x, ic.value, fc.value, it.value

    def set_blocks(self, typ, p, a3, v3):
        """Caller-given residual blocks in place of build_blocks' (ll_set_blocks): typ [M] (0 invalid / 1 line / 2 plane), p [M,4] features (scan
        frame, intensity = time stamp), a3 [M,3] anchors (fp32), v3 [M,3] directions / normals; the state is self.state."""
        t = np.ascontiguousarray(typ, np.int32)
        p = np.ascontiguousarray(p, np.float32)
        a = np.ascontiguousarray(a3, np.float32)
        v = np.ascontiguousarray(v3, np.float64)
        M = t.shape[0]
        assert p.shape == (M, 4) and a.shape == (M, 3) and v.shape == (M, 3)
        self.ctx.check(self.ctx._lib.ll_set_blocks(self.ctx.h, C.byref(self.state), M, t.ctypes.data, p.ctypes.data, a.ctypes.data, v.ctypes.data))
        self._hook_slots = M

    def solve_fused(self, x7, prerun, max_iterations, want_l1=True):
        """One fused ICP iteration of the solver over the resident blocks (ll_solve_fused).  Returns (x, threshold, n_distinct, n_kept, l1 or
        None, (solve #1 iterations, solve #2 iterations))."""
        x = np.array(x7, np.float64)
        thr, nd, nk, it = C.c_double(), C.c_int(), C.c_int(), np.zeros(2, np.int32)
        l1 = np.empty(getattr(self, "_hook_slots", 0)) if want_l1 else None
        self.ctx.check(self.ctx._lib.ll_solve_fused(self.ctx.h, int(prerun), int(max_iterations), x.ctypes.data, C.byref(thr), C.byref(nd), C.byref(nk),
                                                    l1.ctypes.data if want_l1 else None, it.ctypes.data))
        return x, thr.value, nd.value, nk.value, l1, (int(it[0]), int(it[1]))


def register_batch(ctx: Context, match_map: Map, items, states):
    """n (1 ... LL_MAX_BATCH) independent registrations against one map in one call (ll_register_batch): items[i] = (corner, surf) feature
    clouds, states[i] = its capi.RegState.  Items may share a scan.  Returns (results, item_status): item i's RegResult and status are what
    find_out_incremental_transfrom would give for it alone (status LL_OK, or LL_ERR_NO_BLOCKS for an item that would fail alone and dropped
    out); the gpu_ms_* fields of every result time the whole batch.  An error of the whole call (count, sharded map, mixed deblur, capacity)
    raises, with nothing run."""
    n = len(items)
    if len(states) != n:
        raise ValueError("one state per item")
    arrs = [(_pts(c), _pts(s)) for c, s in items]
    fmt = arrs[0][0][1] if arrs else capi.LL_FMT_XYZI16
    if any(c[1] != fmt or s[1] != fmt for c, s in arrs):
        raise ValueError("every cloud of a batch has the same point format")
    corners = (C.c_void_p * max(n, 1))(*[c[0].ctypes.data for c, _ in arrs])
    surfs = (C.c_void_p * max(n, 1))(*[s[0].ctypes.data for _, s in arrs])
    nc = (C.c_size_t * max(n, 1))(*[c[0].shape[0] for c, _ in arrs])
    ns = (C.c_size_t * max(n, 1))(*[s[0].shape[0] for _, s in arrs])
    st = (capi.RegState * max(n, 1))(*states)
    res = (capi.RegResult * max(n, 1))()
    status = (C.c_int * max(n, 1))()
    ctx.check(ctx._lib.ll_register_batch(ctx.h, match_map.h, n, corners, nc, surfs, ns, fmt, capi.LL_HOST, st, res, status))
    return [res[i] for i in range(n)], [int(status[i]) for i in range(n)]


def inlier_select(ctx: Context, l1, ratio: float):
    """compute_inlier_residual_threshold (point_cloud_registration.hpp:153-161) over caller-given L1 norms (ll_inlier_select): the fused solver
    kernel's grid-wide select, as the sharded mode runs it.  Returns (value, number of distinct values); +inf / NaN are skipped."""
    v = np.ascontiguousarray(l1, np.float64)
    out, nd = C.c_double(), C.c_int()
    ctx.check(ctx._lib.ll_inlier_select(ctx.h, v.ctypes.data, v.shape[0], float(ratio), C.byref(out), C.byref(nd)))
    return out.value, nd.value


def scan_to_pose(ctx: Context, match_map: Map, raw, stamp, pipeline: capi.PipelineCfg, state: capi.RegState, where=capi.LL_HOST, n=None, fmt=None):
    """Whole per-scan step: raw scan -> features -> VoxelGrid x2 -> registration (ll_scan_to_pose)."""
    if where == capi.LL_HOST:
        pts, fmt = _pts(raw)
        ptr, n = pts.ctypes.data, pts.shape[0]
    else:
        ptr = int(raw)
    res = capi.RegResult()
    nc, ns = C.c_int(), C.c_int()
    ctx.check(ctx._lib.ll_scan_to_pose(ctx.h, match_map.h, ptr, n, fmt, where, float(stamp), C.byref(pipeline), C.byref(state), C.byref(res), C.byref(nc), C.byref(ns)))
    return res, nc.value, ns.value


def frame_to_pose(ctx: Context, match_map: Map, heads, stamps, pipeline: capi.PipelineCfg, state: capi.RegState, where=capi.LL_HOST, ns=None, fmt=None):
    """Multi-head frame (Mid-100: three Mid-40 heads): one extractor over the heads in turn, feature clouds summed, VoxelGrids, registration
    (ll_frame_to_pose; laser_feature_extractor.hpp:303-380).  heads: list of [n,4] arrays (LL_HOST) or of device pointers (LL_DEVICE, with ns)."""
    k = len(heads)
    if where == capi.LL_HOST:
        arrs = [_pts(h) for h in heads]
        fmt = arrs[0][1]
        ptrs = (C.c_void_p * k)(*[a.ctypes.data for a, _ in arrs])
        sizes = (C.c_size_t * k)(*[a.shape[0] for a, _ in arrs])
    else:
        ptrs = (C.c_void_p * k)(*[int(h) for h in heads])
        sizes = (C.c_size_t * k)(*[int(n) for n in ns])
    st = (C.c_double * k)(*[float(t) for t in stamps])
    res = capi.RegResult()
    nc, nsf = C.c_int(), C.c_int()
    ctx.check(ctx._lib.ll_frame_to_pose(ctx.h, match_map.h, k, ptrs, sizes, fmt, where, st, C.byref(pipeline), C.byref(state), C.byref(res), C.byref(nc), C.byref(nsf)))
    return res, nc.value, nsf.value


def features_to_pointcloud2(ctx: Context, which: int) -> bytes:
    """pcl::toROSMsg of the last registration's corner (0) / surface (1) features, in the layout of Context.set_point_layout (ll_features_to_pointcloud2)."""
    n = C.c_size_t()
    ctx.check(ctx._lib.ll_features_to_pointcloud2(ctx.h, which, None, 0, C.byref(n)))
    step = ctx._layout_step if hasattr(ctx, "_layout_step") else 16
    buf = np.zeros(n.value * step, np.uint8)
    if n.value:
        ctx.check(ctx._lib.ll_features_to_pointcloud2(ctx.h, which, buf.ctypes.data, buf.shape[0], C.byref(n)))
    return buf.tobytes()


def yaw_circle(yaw_step_deg: float, tilt_q=None):
    """Rotations of a yaw circle (n = round(360 / yaw_step_deg) yaws k * step about z, k = 0 ... n - 1), each composed with an optional tilt
    applied first: q_k = q_yaw(k) * tilt_q.  [n, 4] (w, x, y, z), fp64."""
    n = int(round(360.0 / float(yaw_step_deg)))
    if n < 1:
        raise ValueError("yaw_step_deg must be in (0, 360]")
    a = np.radians(np.arange(n) * (360.0 / n)) * 0.5
    q = np.stack([np.cos(a), np.zeros(n), np.zeros(n), np.sin(a)], axis=1)
    if tilt_q is not None:
        b = np.asarray(tilt_q, np.float64)
        b = b / np.linalg.norm(b)
        w1, x1, y1, z1 = q.T
        w2, x2, y2, z2 = b
        q = np.stack([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                      w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2], axis=1)
    return np.ascontiguousarray(q)


def reloc_cfg(rot_wxyz, t0, step, nt, k=8, cyclic=True):
    """(capi.RelocCfg, keepalive) of rotations [n, 4] and the lattice t = t0 + i * step, i in 0 ... nt - 1 per axis."""
    rot = np.ascontiguousarray(rot_wxyz, np.float64).reshape(-1, 4)
    cfg = capi.RelocCfg()
    cfg.n_rot = rot.shape[0]
    cfg.rot_wxyz = rot.ctypes.data_as(C.POINTER(C.c_double))
    cfg.rot_cyclic = int(bool(cyclic))
    cfg.t0[:] = [float(v) for v in t0]
    cfg.step[:] = [float(v) for v in step]
    cfg.nt[:] = [int(v) for v in nt]
    cfg.max_candidates = int(k)
    return cfg, rot


def window_lattice(window):
    """((x0, x1, dx), (y0, y1, dy), (z0, z1, dz)) -> (t0, step, nt): every lattice point t0 + i * step inside [lo, hi] per axis (dz may be 0 for one
    height)."""
    t0, step, nt = [], [], []
    for lo, hi, d in window:
        n = 1 if d == 0 or hi == lo else int(np.floor((hi - lo) / d + 1e-9)) + 1
        t0.append(float(lo)); step.append(float(d) if d else 1.0); nt.append(n)
    return t0, step, nt


class RelocIndex:
    """The occupancy index of a map for relocalization (ll_reloc_index_build): the map's own clouds voxelised at `res`, dilated by `dilate`
    voxels (Chebyshev), with the buffers of up to max_hypotheses hypotheses allocated once."""

    def __init__(self, ctx: Context, match_map: Map, res: float = 0.2, dilate: int = 1, max_hypotheses: int = 1 << 20):
        self.ctx, self.map = ctx, match_map
        h = C.c_void_p()
        ctx.check(ctx._lib.ll_reloc_index_build(ctx.h, match_map.h, float(res), int(dilate), int(max_hypotheses), C.byref(h)))
        self.h = h

    def read(self):
        """(dims [3] int, lo [3] float32, words uint32): the bitmask, voxel x + dims0 (y + dims1 z) in bit v & 31 of word v >> 5."""
        dims, lo = np.zeros(3, np.int32), np.zeros(3, np.float32)
        st = self.ctx._lib.ll_reloc_index_read(self.h, dims.ctypes.data, lo.ctypes.data, None, 0)
        if st != capi.LL_OK:
            raise LoamLivoxError(f"ll_reloc_index_read: status {st}")
        words = np.zeros((int(np.prod(dims.astype(np.int64))) + 31) // 32, np.uint32)
        st = self.ctx._lib.ll_reloc_index_read(self.h, dims.ctypes.data, lo.ctypes.data, words.ctypes.data, words.shape[0])
        if st != capi.LL_OK:
            raise LoamLivoxError(f"ll_reloc_index_read: status {st}")
        return dims, lo, words

    def close(self):
        if getattr(self, "h", None):
            self.ctx._lib.ll_reloc_index_release(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def reloc_scores(ctx: Context, index: RelocIndex, score_pts, rot_wxyz, t0, step, nt, cyclic=True):
    """The score of every hypothesis (ll_reloc_scores), int32 in hypothesis order h = i + nt0 (j + nt1 (k + nt2 r))."""
    p, fmt = _pts(score_pts)
    cfg, _keep = reloc_cfg(rot_wxyz, t0, step, nt, 1, cyclic)
    out = np.zeros(cfg.n_rot * int(np.prod(nt)), np.int32)
    ctx.check(ctx._lib.ll_reloc_scores(ctx.h, index.h, p.ctypes.data, p.shape[0], fmt, capi.LL_HOST, C.byref(cfg), out.ctypes.data))
    return out


def _features(corners, surfs):
    """(corners, surfaces, their one point format) of relocalize and relocalize_field."""
    c, fmt = _pts(corners)
    s, fmt2 = _pts(surfs)
    if fmt != fmt2:
        raise ValueError("corners and surfaces in one point format")
    return c, s, fmt


def _coarse_args(state, yaw_step_deg, tilt_q, window, k):
    """(`state` or capi.default_reg_state past the initialisation gate, the coarse capi.RelocCfg of the yaw circle and the window's lattice,
    its keepalive) of relocalize and relocalize_field."""
    if state is None:
        state = capi.default_reg_state()
        state.current_frame_index = state.mapping_init_accumulate_frames + 1
    rot = yaw_circle(yaw_step_deg, tilt_q)
    t0, step, nt = window_lattice(window)
    cfg, keep = reloc_cfg(rot, t0, step, nt, k, cyclic=True)
    return state, cfg, keep


def relocalize(ctx: Context, match_map: Map, index: RelocIndex, corners, surfs, score_leaf: float = 0.5, window=((-1.0, 1.0, 1.0), (-1.0, 1.0, 1.0), (0.0, 0.0, 0.0)),
               yaw_step_deg: float = 10.0, tilt_q=None, k: int = 8, state: capi.RegState | None = None, score_pts=None):
    """Find the pose of a scan (its scan-frame corner / surface features) in `match_map` without an initial guess (ll_relocalize).

    The score points are a VoxelGrid of both feature clouds at score_leaf (through the library), unless score_pts is given.  The hypotheses are a
    yaw circle of yaw_step_deg (composed with tilt_q, the sensor's roll / pitch, when given) times the translation lattice of `window`
    (((x0, x1, dx), (y0, y1, dy), (z0, z1, dz))).  The first k peaks of the score are refined by the batched registration with `state` (default:
    capi.default_reg_state past the initialisation gate).  Returns {"candidates": [{hypothesis, score, q, t}], "refined": [RegResult],
    "item_status": [int], "best": rank or -1, "n_score": int}."""
    c, s, fmt = _features(corners, surfs)
    if score_pts is None:
        both = np.concatenate([c[:, :4], s[:, :4]] if fmt == capi.LL_FMT_XYZI16 else [c[:, [0, 1, 2, 4]], s[:, [0, 1, 2, 4]]], axis=0)
        score_pts = voxel_grid_filter(ctx, both, float(score_leaf))
    sp, sfmt = _pts(score_pts)
    if sfmt != fmt:
        sp = np.ascontiguousarray(sp[:, [0, 1, 2, 4]] if sfmt == capi.LL_FMT_PCL32 else np.concatenate([sp, np.zeros((sp.shape[0], 4), np.float32)], axis=1))
    state, cfg, _keep = _coarse_args(state, yaw_step_deg, tilt_q, window, k)
    K = int(k)
    cand, res, status = (capi.RelocCandidate * K)(), (capi.RegResult * K)(), (C.c_int * K)()
    n, best = C.c_int(), C.c_int()
    ctx.check(ctx._lib.ll_relocalize(ctx.h, match_map.h, index.h, sp.ctypes.data, sp.shape[0], c.ctypes.data, c.shape[0], s.ctypes.data, s.shape[0], fmt, capi.LL_HOST,
                                     C.byref(cfg), C.byref(state), cand, res, status, C.byref(n), C.byref(best)))
    cands = [{"hypothesis": int(cand[i].hypothesis), "score": int(cand[i].score), "q": np.array(cand[i].q_wxyz), "t": np.array(cand[i].t)} for i in range(n.value)]
    return {"candidates": cands, "refined": [res[i] for i in range(n.value)], "item_status": [int(status[i]) for i in range(n.value)], "best": int(best.value),
            "n_score": int(sp.shape[0])}


class RelocField:
    """The class-aware distance fields of a map for relocalization (ll_reloc_field_build): per class, the squared voxel distance at `res` to the
    class's nearest map point, truncated at trunc^2, with the buffers of up to max_hypotheses hypotheses allocated once.  The defaults (0.2 m,
    T = 2) are the setting that found every measured case (DESIGN.md §4.3.1)."""

    def __init__(self, ctx: Context, match_map: Map, res: float = 0.2, trunc: int = 2, max_hypotheses: int = 1 << 20):
        self.ctx, self.map = ctx, match_map
        h = C.c_void_p()
        ctx.check(ctx._lib.ll_reloc_field_build(ctx.h, match_map.h, float(res), int(trunc), int(max_hypotheses), C.byref(h)))
        self.h = h

    def read(self, which: int):
        """(dims [3] int, lo [3] float32, d2 uint8 [dims2, dims1, dims0]): the field of class `which` (0 corner, 1 surface)."""
        dims, lo = np.zeros(3, np.int32), np.zeros(3, np.float32)
        st = self.ctx._lib.ll_reloc_field_read(self.h, int(which), dims.ctypes.data, lo.ctypes.data, None, 0)
        if st != capi.LL_OK:
            raise LoamLivoxError(f"ll_reloc_field_read: status {st}")
        d2 = np.zeros((int(dims[2]), int(dims[1]), int(dims[0])), np.uint8)
        st = self.ctx._lib.ll_reloc_field_read(self.h, int(which), dims.ctypes.data, lo.ctypes.data, d2.ctypes.data, d2.size)
        if st != capi.LL_OK:
            raise LoamLivoxError(f"ll_reloc_field_read: status {st}")
        return dims, lo, d2

    def close(self):
        if getattr(self, "h", None):
            self.ctx._lib.ll_reloc_field_release(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def fine_cfg(rot_wxyz, step, nt):
    """(capi.RelocFineCfg, keepalive) of rotation offsets [n, 4] and the odd lattice nt x step centred on each candidate."""
    rot = np.ascontiguousarray(rot_wxyz, np.float64).reshape(-1, 4)
    cfg = capi.RelocFineCfg()
    cfg.n_rot = rot.shape[0]
    cfg.rot_wxyz = rot.ctypes.data_as(C.POINTER(C.c_double))
    cfg.step[:] = [float(v) for v in step]
    cfg.nt[:] = [int(v) for v in nt]
    return cfg, rot


def fine_search(yaw_step_deg: float, window, fine_yaw_step_deg: float = 1.0, fine_t_step: float = 0.1, fine_t_half: float = 1.5):
    """The fine search of a coarse yaw circle and window: yaw offsets of +-half the coarse yaw step at fine_yaw_step_deg, and on every axis the
    window steps along, +-fine_t_half coarse steps at fine_t_step (one point on an axis of one height).  Returns (dq [n, 4], step [3], nt [3]).
    Half a coarse step is not enough: at a yaw 4.5 deg off, the coarse peaks of the C2 room lie about 1.5 m to either side of the truth
    (DESIGN.md §4.3.1)."""
    ny = int(np.floor(0.5 * float(yaw_step_deg) / float(fine_yaw_step_deg) + 1e-9))
    a = np.radians(np.arange(-ny, ny + 1) * float(fine_yaw_step_deg)) * 0.5
    dq = np.ascontiguousarray(np.stack([np.cos(a), np.zeros_like(a), np.zeros_like(a), np.sin(a)], axis=1))
    _, coarse_step, coarse_nt = window_lattice(window)
    nt = [1 if n == 1 else 2 * int(np.floor(float(fine_t_half) * d / float(fine_t_step) + 1e-9)) + 1 for d, n in zip(coarse_step, coarse_nt)]
    return dq, [float(fine_t_step)] * 3, nt


def _score_pair(fmt, score_corner, score_surf):
    c, cf = _pts(score_corner)
    s, sf = _pts(score_surf)
    if cf != fmt or sf != fmt:
        raise ValueError("score points in the features' point format")
    return c, s


def reloc_field_scores(ctx: Context, field: RelocField, score_corner, score_surf, rot_wxyz, t0, step, nt):
    """The field score of every hypothesis (ll_reloc_field_scores), int32 in hypothesis order h = i + nt0 (j + nt1 (k + nt2 r))."""
    c, s = _score_pair(_pts(score_corner)[1], score_corner, score_surf)
    fmt = _pts(c)[1]
    cfg, _keep = reloc_cfg(rot_wxyz, t0, step, nt, 1)
    out = np.zeros(cfg.n_rot * int(np.prod(nt)), np.int32)
    ctx.check(ctx._lib.ll_reloc_field_scores(ctx.h, field.h, c.ctypes.data, c.shape[0], s.ctypes.data, s.shape[0], fmt, capi.LL_HOST, C.byref(cfg), out.ctypes.data))
    return out


def relocalize_field(ctx: Context, match_map: Map, field: RelocField, corners, surfs, score_leaf: float = 0.5,
                     window=((-1.0, 1.0, 1.0), (-1.0, 1.0, 1.0), (0.0, 0.0, 0.0)), yaw_step_deg: float = 10.0, tilt_q=None, k: int = 8,
                     state: capi.RegState | None = None, score_pts=None, fine_yaw_step_deg: float = 1.0, fine_t_step: float = 0.1,
                     fine_t_half: float = 1.5):
    """Find the pose of a scan (its scan-frame corner / surface features) in `match_map` without an initial guess (ll_relocalize_field).

    The score points are each class's VoxelGrid at score_leaf (through the library), unless score_pts = (corner, surface) is given.  The coarse
    hypotheses are those of `relocalize`; every one of the first k peaks gets the fine search of `fine_search` around it, the best fine hypothesis
    of each is refined by the batched registration with `state`, and the accepted item of the largest field score at its refined pose wins.
    Returns {"candidates": [{hypothesis, score, q, t, fine_index, fine_score, fine_q, fine_t, verify_score}], "refined": [RegResult],
    "item_status": [int], "best": rank or -1, "n_score": (corner, surface)}."""
    c, s, fmt = _features(corners, surfs)
    if score_pts is None:
        score_pts = (voxel_grid_filter(ctx, c, float(score_leaf)), voxel_grid_filter(ctx, s, float(score_leaf)))
        if fmt == capi.LL_FMT_PCL32:
            score_pts = tuple(np.concatenate([p, np.zeros((p.shape[0], 4), np.float32)], axis=1) for p in score_pts)
    sc, ss = _score_pair(fmt, *score_pts)
    state, cfg, _keep = _coarse_args(state, yaw_step_deg, tilt_q, window, k)
    dq, fstep, fnt = fine_search(yaw_step_deg, window, fine_yaw_step_deg, fine_t_step, fine_t_half)
    fcfg, _keep2 = fine_cfg(dq, fstep, fnt)
    K = int(k)
    cand, res, status = (capi.RelocFieldCandidate * K)(), (capi.RegResult * K)(), (C.c_int * K)()
    n, best = C.c_int(), C.c_int()
    ctx.check(ctx._lib.ll_relocalize_field(ctx.h, match_map.h, field.h, sc.ctypes.data, sc.shape[0], ss.ctypes.data, ss.shape[0], c.ctypes.data, c.shape[0],
                                           s.ctypes.data, s.shape[0], fmt, capi.LL_HOST, C.byref(cfg), C.byref(fcfg), C.byref(state), cand, res, status,
                                           C.byref(n), C.byref(best)))
    cands = [{"hypothesis": int(x.hypothesis), "score": int(x.score), "q": np.array(x.q_wxyz), "t": np.array(x.t), "fine_index": int(x.fine_index),
              "fine_score": int(x.fine_score), "fine_q": np.array(x.fine_q_wxyz), "fine_t": np.array(x.fine_t), "verify_score": int(x.verify_score)}
             for x in (cand[i] for i in range(n.value))]
    return {"candidates": cands, "refined": [res[i] for i in range(n.value)], "item_status": [int(status[i]) for i in range(n.value)], "best": int(best.value),
            "n_score": (int(sc.shape[0]), int(ss.shape[0]))}


class Scene_alignment:
    """Mirror of Scene_alignment::find_tranfrom_of_two_mappings from the point where the four feature clouds exist
    (loam_livox/source/scene_alignment.hpp:269-353): coarse-to-fine registration of keyframe b's features onto keyframe a's."""

    def __init__(self, ctx: Context, line_res: float = 0.4, plane_res: float = 0.4, **kw):
        self.ctx = ctx
        self.cfg = capi.AlignCfg()
        ctx._lib.ll_align_cfg_default(C.byref(self.cfg))
        self.cfg.line_res, self.cfg.plane_res = line_res, plane_res
        for k, v in kw.items():
            setattr(self.cfg, k, v)

    def find_tranfrom_of_two_mappings(self, source_line, source_plane, target_line, target_plane, t_init=(0.0, 0.0, 0.0)):
        sl, fmt = _pts(source_line)
        sp, _ = _pts(source_plane)
        tl, _ = _pts(target_line)
        tp, _ = _pts(target_plane)
        self.cfg.t_init[:] = list(t_init)
        res, runs = capi.RegResult(), C.c_int()
        self.ctx.check(self.ctx._lib.ll_scene_align(self.ctx.h, sl.ctypes.data, sl.shape[0], sp.ctypes.data, sp.shape[0], tl.ctypes.data, tl.shape[0], tp.ctypes.data, tp.shape[0],
                                                    fmt, capi.LL_HOST, C.byref(self.cfg), C.byref(res), C.byref(runs)))
        self.m_q_w_curr, self.m_t_w_curr = np.array(res.q_w_curr), np.array(res.t_w_curr)
        self.scales_run = runs.value
        return res

    def align_keyframes(self, keyframe_a: "Keyframe", keyframe_b: "Keyframe"):
        """find_tranfrom_of_two_mappings(keyframe_a, keyframe_b) on the keyframes' device-resident typed clouds (scene_alignment.hpp:275-303):
        source = a's line / plane cells, target = b's, t_init = (a.get_center() - b.get_center()) in float, then double."""
        sl, nsl = keyframe_a.device_cloud(capi.LL_CELL_LINE)
        sp, nsp = keyframe_a.device_cloud(capi.LL_CELL_PLANE)
        tl, ntl = keyframe_b.device_cloud(capi.LL_CELL_LINE)
        tp, ntp = keyframe_b.device_cloud(capi.LL_CELL_PLANE)
        self.cfg.t_init[:] = [float(v) for v in (keyframe_a.get_center() - keyframe_b.get_center()).astype(np.float32)]
        res, runs = capi.RegResult(), C.c_int()
        self.ctx.check(self.ctx._lib.ll_scene_align(self.ctx.h, sl, nsl, sp, nsp, tl, ntl, tp, ntp, capi.LL_FMT_XYZI16, capi.LL_DEVICE, C.byref(self.cfg),
                                                    C.byref(res), C.byref(runs)))
        self.m_q_w_curr, self.m_t_w_curr = np.array(res.q_w_curr), np.array(res.t_w_curr)
        self.scales_run = runs.value
        return res


def pg_edges(id_begin, id_end, q_wxyz, t, information=None):
    """An array of capi.PgEdge (Ceres_pose_graph_3d::Constraint3d): information defaults to the identity, as the reference always passes."""
    id_begin, id_end = np.atleast_1d(id_begin), np.atleast_1d(id_end)
    q, t = np.asarray(q_wxyz, np.float64).reshape(-1, 4), np.asarray(t, np.float64).reshape(-1, 3)
    W = np.broadcast_to(np.eye(6) if information is None else np.asarray(information, np.float64), (len(id_begin), 6, 6))
    out = (capi.PgEdge * len(id_begin))()
    for k in range(len(id_begin)):
        out[k].id_begin, out[k].id_end = int(id_begin[k]), int(id_end[k])
        out[k].q_wxyz[:], out[k].t[:], out[k].information[:] = list(q[k]), list(t[k]), list(W[k].reshape(36))
    return out


def pg_loop_edge(icp_q_wxyz, icp_t, pose_a, id_a: int, pose_b, id_b: int) -> capi.PgEdge:
    """Scene_alignment::add_constrain_of_loop on the pose ll_scene_align returned (laser_mapping.hpp:1062-1078): a = the older keyframe
    (id_end), b = the newer one (id_begin); poses as (q_wxyz, t) rows of 7."""
    e = capi.PgEdge()
    pa, pb = capi.Pose(), capi.Pose()
    pa.q_wxyz[:], pa.t[:] = list(pose_a[:4]), list(pose_a[4:7])
    pb.q_wxyz[:], pb.t[:] = list(pose_b[:4]), list(pose_b[4:7])
    q, t = np.ascontiguousarray(icp_q_wxyz, np.float64), np.ascontiguousarray(icp_t, np.float64)
    capi.lib().ll_pose_graph_loop_edge(q.ctypes.data, t.ctypes.data, C.byref(pa), id_a, C.byref(pb), id_b, C.byref(e))
    return e


def keyframes_repose(ctx: Context, clouds, poses_ori, poses_opt, leaf: float):
    """Mapping_refine::refine_pointcloud (ceres_pose_graph_3d.hpp:437-500, if_save == 0) for every keyframe: clouds is a list of [n_k, 4] arrays,
    poses rows of 7 (q_wxyz, t) before / after the optimization.  Returns the list of re-posed, down-sampled clouds (intensity 0)."""
    arrs = [np.ascontiguousarray(c, np.float32).reshape(-1, 4) for c in clouds]
    allp = np.concatenate(arrs) if arrs else np.zeros((0, 4), np.float32)
    allp = np.ascontiguousarray(allp)
    ends = np.cumsum([a.shape[0] for a in arrs]).astype(np.uint64)
    po, pp = np.ascontiguousarray(poses_ori, np.float64).reshape(-1, 7), np.ascontiguousarray(poses_opt, np.float64).reshape(-1, 7)
    out, cnt = np.zeros((max(allp.shape[0], 1), 4), np.float32), np.zeros(len(arrs), np.uint64)
    ctx.check(ctx._lib.ll_keyframes_repose(ctx.h, allp.ctypes.data, allp.shape[0], ends.ctypes.data, len(arrs), po.ctypes.data, pp.ctypes.data, leaf,
                                           out.ctypes.data, cnt.ctypes.data))
    res, w = [], 0
    for c in cnt:
        res.append(out[w:w + int(c)].copy())
        w += int(c)
    return res


class PoseGraph:
    """Mirror of Ceres_pose_graph_3d::pose_graph_optimization (ceres_pose_graph_3d.hpp:282-352) on the device.  Poses are an [n, 7] array of
    rows (qw, qx, qy, qz, tx, ty, tz), keyframe order; pose 0 is held constant."""

    def __init__(self, ctx: Context, reserve_nodes: int = 1024, reserve_edges: int = 2048):
        self.ctx = ctx
        h = C.c_void_p()
        ctx.check(ctx._lib.ll_pose_graph_create(ctx.h, reserve_nodes, reserve_edges, C.byref(h)))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.ctx._lib.ll_pose_graph_release(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def optimize(self, poses, edges, max_iterations: int = 200):
        """Returns (optimized poses, capi.PgSummary); `poses` is not modified."""
        x = np.ascontiguousarray(poses, np.float64).reshape(-1, 7).copy()
        s = capi.PgSummary()
        self.ctx.check(self.ctx._lib.ll_pose_graph_optimize(self.h, x.ctypes.data, x.shape[0], C.cast(edges, C.c_void_p) if len(edges) else None, len(edges),
                                                            max_iterations, C.byref(s)))
        return x, s

    def step(self, poses, edges, radius: float):
        """The LM step solve at `poses` (ll_pose_graph_step): (cost, gradient [n,6], scaling [n,6], step [n,6], valid)."""
        x = np.ascontiguousarray(poses, np.float64).reshape(-1, 7)
        n = x.shape[0]
        g, s, st = np.zeros((n, 6)), np.zeros((n, 6)), np.zeros((n, 6))
        cost, valid = C.c_double(), C.c_int()
        self.ctx.check(self.ctx._lib.ll_pose_graph_step(self.h, x.ctypes.data, n, C.cast(edges, C.c_void_p), len(edges), radius, C.byref(cost), g.ctypes.data,
                                                        s.ctypes.data, st.ctypes.data, C.byref(valid)))
        return cost.value, g, s, st, bool(valid.value)


class Points_cloud_map:
    """Device-resident voxel-cell map as the matching path uses it (Points_cloud_map<float>, loam_livox/source/cell_map_keyframe.hpp:264;
    append_cloud :619, find_cells_in_radius :761; the consumer is update_buff_for_matching, loam_livox/source/laser_mapping.hpp:471-516)."""

    def __init__(self, ctx: Context, resolution: float = 1.0, revisit_threshold: int = 2000, max_cells: int = 0):
        self.ctx = ctx
        h = C.c_void_p()
        ctx.check(ctx._lib.ll_cellmap_create(ctx.h, float(resolution), int(revisit_threshold), int(max_cells), C.byref(h)))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.ctx._lib.ll_cellmap_release(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reserve(self, store_points: int, scan_points: int = 0):
        """Allocate now for that many stored points (and appends of up to scan_points): nothing is reallocated below that."""
        self.ctx.check(self.ctx._lib.ll_cellmap_reserve(self.ctx.h, self.h, int(store_points), int(scan_points)))

    def append_cloud(self, pts):
        pts, fmt = _pts(pts)
        self.ctx.check(self.ctx._lib.ll_cellmap_append(self.ctx.h, self.h, pts.ctypes.data, pts.shape[0], fmt, capi.LL_HOST))

    def stats(self):
        c, p, f = C.c_int(), C.c_int(), C.c_int()
        self.ctx.check(self.ctx._lib.ll_cellmap_stats(self.ctx.h, self.h, C.byref(c), C.byref(p), C.byref(f)))
        return c.value, p.value, f.value

    def get_cells_size(self) -> int:
        return self.stats()[0]

    def assemble(self, q_w_curr, t_w_curr, search_range=100.0, fov_angle=45.0, leaf=0.4, replace=True):
        """cells in radius + if_pt_in_fov + per-cell VoxelGrid (+ replace) -> (n x 4 float32 cloud, cells in the FOV)."""
        q = np.ascontiguousarray(q_w_curr, np.float64)
        t = np.ascontiguousarray(t_w_curr, np.float64)
        cap = max(self.stats()[1], 1)
        out = np.empty((cap, 4), np.float32)
        n, nf, dev = C.c_size_t(), C.c_int(), C.c_void_p()
        self.ctx.check(self.ctx._lib.ll_cellmap_assemble(self.ctx.h, self.h, q.ctypes.data, t.ctypes.data, float(search_range), float(fov_angle), float(leaf), int(bool(replace)),
                                                         out.ctypes.data, cap, C.byref(n), C.byref(nf), C.byref(dev)))
        return out[:n.value].copy(), nf.value


class Keyframe:
    """Maps_keyframe<float> over the cells of a full-resolution Points_cloud_map (loam_livox/source/cell_map_keyframe.hpp:1002-1494): cells
    from append (laser_mapping.hpp:1527-1533), analyze() for the types, centre, ROI range and feature images, the typed clouds on the device."""

    def __init__(self, ctx: Context):
        self.ctx = ctx
        h = C.c_void_p()
        ctx.check(ctx._lib.ll_keyframe_create(ctx.h, C.byref(h)))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.ctx._lib.ll_keyframe_release(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def append(ctx: Context, cellmap: "Points_cloud_map", pts, open_keyframes):
        """append_cloud(pts, &cell_vec) on the cell map, then add_cells(cell_vec) on every open keyframe."""
        pts, fmt = _pts(pts)
        hs = (C.c_void_p * max(len(open_keyframes), 1))(*[k.h for k in open_keyframes])
        ctx.check(ctx._lib.ll_keyframe_append(ctx.h, cellmap.h, pts.ctypes.data, pts.shape[0], fmt, capi.LL_HOST, hs, len(open_keyframes)))

    def analyze(self, cellmap: "Points_cloud_map", incremental_cov: bool = False) -> capi.KeyframeInfo:
        info = capi.KeyframeInfo()
        self.ctx.check(self.ctx._lib.ll_keyframe_analyze(self.ctx.h, cellmap.h, self.h, int(bool(incremental_cov)), C.byref(info)))
        return info

    def info(self) -> capi.KeyframeInfo:
        info = capi.KeyframeInfo()
        if self.ctx._lib.ll_keyframe_get_info(self.h, C.byref(info)) != capi.LL_OK:
            raise LoamLivoxError("keyframe not analyzed since its last append")
        return info

    def get_center(self):
        return np.array(self.info().center, np.float32)

    def cells(self, analyzed: bool = True):
        """(keys uint64, incarnations, types, feature vectors [n, 3]) in the keyframe's cell order; types / vectors need an analysis."""
        n = C.c_int()
        self.ctx.check(self.ctx._lib.ll_keyframe_cells(self.ctx.h, self.h, None, None, None, None, 0, C.byref(n)))
        k, e = np.zeros(n.value, np.uint64), np.zeros(n.value, np.int32)
        t, v = np.zeros(n.value, np.int32), np.zeros((n.value, 3), np.float32)
        self.ctx.check(self.ctx._lib.ll_keyframe_cells(self.ctx.h, self.h, k.ctypes.data, e.ctypes.data, t.ctypes.data if analyzed else None,
                                                       v.ctypes.data if analyzed else None, n.value, C.byref(n)))
        return k, e, t, v

    def images(self):
        """[4, 60, 60]: line counts, plane counts (before the blur), blurred line image, blurred plane image."""
        out = np.zeros((4, 60, 60), np.float32)
        self.ctx.check(self.ctx._lib.ll_keyframe_images(self.ctx.h, self.h, *[out[i].ctypes.data for i in range(4)]))
        return out

    def extract_specify_points(self, which: int):
        """which = capi.LL_CELL_LINE / LL_CELL_PLANE / LL_CELL_ALL -> n x 4 float32 (intensity 0)."""
        n, dev = C.c_size_t(), C.c_void_p()
        self.ctx.check(self.ctx._lib.ll_keyframe_cloud(self.ctx.h, self.h, which, None, 0, C.byref(n), C.byref(dev)))
        out = np.zeros((n.value, 4), np.float32)
        self.ctx.check(self.ctx._lib.ll_keyframe_cloud(self.ctx.h, self.h, which, out.ctypes.data, n.value, C.byref(n), C.byref(dev)))
        return out

    def get_all_pointcloud(self):
        return self.extract_specify_points(capi.LL_CELL_ALL)

    def device_cloud(self, which: int):
        """(device pointer, point count) of a typed cloud, for ll_scene_align with LL_DEVICE."""
        n, dev = C.c_size_t(), C.c_void_p()
        self.ctx.check(self.ctx._lib.ll_keyframe_cloud(self.ctx.h, self.h, which, None, 0, C.byref(n), C.byref(dev)))
        return dev.value, n.value


def loop_search(ctx: Context, keyframes, newest: int = -1, cfg: capi.LoopCfg = None):
    """service_loop_detection's candidate search (laser_mapping.hpp:988-1033) for keyframes[newest] against every earlier keyframe:
    (sim_plane [newest], sim_line [newest], candidate indices ascending)."""
    n = len(keyframes)
    newest = n - 1 if newest < 0 else newest
    cfg = cfg if cfg is not None else capi.default_loop_cfg()
    hs = (C.c_void_p * max(n, 1))(*[k.h for k in keyframes])
    sp, sl, cand = np.zeros(max(newest, 1), np.float32), np.zeros(max(newest, 1), np.float32), np.zeros(max(newest, 1), np.int32)
    nc = C.c_int()
    ctx.check(ctx._lib.ll_loop_search(ctx.h, hs, n, newest, C.byref(cfg), sp.ctypes.data, sl.ctypes.data, cand.ctypes.data, C.byref(nc)))
    return sp[:newest], sl[:newest], cand[:nc.value].tolist()


class SequenceError(LoamLivoxError):
    """An error that stopped process_new_frames / process_new_scans at input `done`: `results` holds what completed (per frame, the frames
    before `done` and the pieces of frame `done` completed; per scan, the scans before `done`).  The mapper stands as after the one-by-one calls
    up to and including the failing input, so the caller can go on from input done + 1."""

    def __init__(self, status, message, done, results):
        super().__init__(f"status {status}: {message} (input {done})")
        self.status, self.done, self.results = status, done, results


class Laser_mapping:
    """Streaming odometry: one call per raw scan (Laser_mapping::process_new_scan, loam_livox/source/laser_mapping.hpp:1316-1521, with the
    match-map refresh of update_buff_for_matching :460-566 in matching_mode 1).  All state stays on the device."""

    def __init__(self, ctx: Context, **kw):
        self.ctx = ctx
        cfg = capi.MapperConfig()
        ctx._lib.ll_mapper_config_default(C.byref(cfg))
        reg = kw.pop("reg", None)
        pipeline = kw.pop("pipeline", None)
        if reg is not None:
            cfg.reg = reg
        if pipeline is not None:
            cfg.pipeline = pipeline
        for k, v in kw.items():
            if not hasattr(cfg, k):
                raise AttributeError(k)
            setattr(cfg, k, v)
        self.cfg = cfg
        h = C.c_void_p()
        ctx.check(ctx._lib.ll_mapper_create(ctx.h, C.byref(cfg), C.byref(h)))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.ctx._lib.ll_mapper_release(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def process_new_scan(self, raw, stamp, where=capi.LL_HOST, n=None, fmt=None):
        ptrs, sizes, fmt, _keep = self._clouds([raw], where, None if n is None else [n], fmt)
        res, stats = capi.RegResult(), capi.MapperStats()
        self.ctx.check(self.ctx._lib.ll_mapper_process_scan(self.h, ptrs[0], sizes[0], fmt, where, float(stamp), C.byref(res), C.byref(stats)))
        return res, stats

    def process_new_frame(self, heads, stamps, odom_mode=1, where=capi.LL_HOST, ns=None, fmt=None):
        """One sensor frame (a list of raw clouds, one per head; Mid-100: 3) cut into pieces, every piece registered as a scan of its own
        (odom_mode 1, the shipped configs; 0: piece 0 only).  Returns a list of (RegResult, MapperStats), one per published piece."""
        k = len(heads)
        ptrs, sizes, fmt, _keep = self._clouds(heads, where, ns, fmt)
        st = (C.c_double * k)(*[float(t) for t in stamps])
        cap = capi.LL_MAX_PIECES_PER_FRAME
        res, stats, n = (capi.RegResult * cap)(), (capi.MapperStats * cap)(), C.c_int()
        self.ctx.check(self.ctx._lib.ll_mapper_process_frame(self.h, k, ptrs, sizes, fmt, where, st, int(odom_mode), res, stats, cap, C.byref(n)))
        return [(res[i], stats[i]) for i in range(n.value)]

    @staticmethod
    def _clouds(clouds, where, ns, fmt):
        """(void* array, size_t array, fmt, keepalive) of host clouds ([n,4] / [n,8] float32, or LL_FMT_STRIDED records with ns given) or of
        device pointers (ns given)."""
        if where == capi.LL_HOST and fmt != capi.LL_FMT_STRIDED:
            arrs = [_pts(c) for c in clouds]
            fmt = arrs[0][1] if arrs else capi.LL_FMT_XYZI16
            keep = [a for a, _ in arrs]
            ptrs, sizes = [a.ctypes.data for a in keep], [a.shape[0] for a in keep]
        elif where == capi.LL_HOST:
            keep = [np.ascontiguousarray(c) for c in clouds]
            ptrs, sizes = [a.ctypes.data for a in keep], [int(n) for n in ns]
        else:
            keep, ptrs, sizes = None, [int(c) for c in clouds], [int(n) for n in ns]
        k = len(ptrs)
        return (C.c_void_p * k)(*ptrs), (C.c_size_t * k)(*sizes), fmt, keep

    def process_new_frames(self, frames, stamps, odom_mode=1, where=capi.LL_HOST, ns=None, fmt=None):
        """Several sensor frames in one call (frames[f]: the head clouds of frame f, the same number of heads in every frame; stamps[f]: their
        time stamps; ns[f]: their sizes for device pointers): the results of process_new_frame on each frame in turn, while the front end of
        frame f + 1 runs on the device under the registrations of frame f.  For recorded data; a live node keeps process_new_frame.
        Returns one list of (RegResult, MapperStats) per frame."""
        nf, nh = len(frames), len(frames[0])
        assert all(len(f) == nh for f in frames) and len(stamps) == nf
        flat_ns = [n for f in ns for n in f] if ns is not None else None
        ptrs, sizes, fmt, _keep = self._clouds([h for f in frames for h in f], where, flat_ns, fmt)
        st = (C.c_double * (nf * nh))(*[float(t) for f in stamps for t in f])
        cap = capi.LL_MAX_PIECES_PER_FRAME
        res, stats = (capi.RegResult * (nf * cap))(), (capi.MapperStats * (nf * cap))()
        n_pieces, done = (C.c_int * nf)(), C.c_int()
        status = self.ctx._lib.ll_mapper_process_frames(self.h, nf, nh, ptrs, sizes, fmt, where, st, int(odom_mode), res, stats, cap, n_pieces, C.byref(done))
        out = [[(res[f * cap + i], stats[f * cap + i]) for i in range(n_pieces[f])] for f in range(nf)]
        if status != capi.LL_OK:   # frames before `done` complete, frame `done` up to its failing piece
            raise SequenceError(status, self.ctx._lib.ll_last_error(self.ctx.h).decode(), done.value, out[:done.value + 1] if done.value < nf else out)
        return out

    def process_new_scans(self, raws, stamps, where=capi.LL_HOST, ns=None, fmt=None):
        """Several raw scans in one call: the results of process_new_scan on each in turn, the front end of scan k + 1 running on the device
        under the mapper step of scan k.  Returns one (RegResult, MapperStats) per scan."""
        k = len(raws)
        ptrs, sizes, fmt, _keep = self._clouds(raws, where, ns, fmt)
        st = (C.c_double * k)(*[float(t) for t in stamps])
        res, stats, done = (capi.RegResult * k)(), (capi.MapperStats * k)(), C.c_int()
        status = self.ctx._lib.ll_mapper_process_scans(self.h, k, ptrs, sizes, fmt, where, st, res, stats, C.byref(done))
        if status != capi.LL_OK:
            raise SequenceError(status, self.ctx._lib.ll_last_error(self.ctx.h).decode(), done.value, [(res[i], stats[i]) for i in range(done.value)])
        return [(res[i], stats[i]) for i in range(k)]

    def process_new_sweep(self, front: "Laser_feature", raw, where=capi.LL_HOST, n=None, fmt=None):
        """One spinning-lidar sweep (ll_mapper_process_sweep): the Velodyne front end of `front` (a Laser_feature on this mapper's context),
        less sharp -> corners, less flat -> surfaces, the full cloud's largest intensity -> max_t, then the mapper step, as the reference's
        remapped pipeline runs.  Afterwards front.cloud(k) gives the sweep's five clouds.  Returns (RegResult, MapperStats)."""
        ptrs, sizes, fmt, _keep = self._clouds([raw], where, None if n is None else [n], fmt)
        res, stats = capi.RegResult(), capi.MapperStats()
        self.ctx.check(self.ctx._lib.ll_mapper_process_sweep(self.h, front.h, ptrs[0], sizes[0], fmt, where, C.byref(res), C.byref(stats)))
        return res, stats

    def process_new_sweeps(self, front: "Laser_feature", raws, where=capi.LL_HOST, ns=None, fmt=None):
        """Several sweeps in one call: the results of process_new_sweep on each in turn, the front end of sweep k + 1 running on the device
        under the mapper step of sweep k.  Returns one (RegResult, MapperStats) per sweep; an error raises SequenceError."""
        k = len(raws)
        ptrs, sizes, fmt, _keep = self._clouds(raws, where, ns, fmt)
        res, stats, done = (capi.RegResult * k)(), (capi.MapperStats * k)(), C.c_int()
        status = self.ctx._lib.ll_mapper_process_sweeps(self.h, front.h, k, ptrs, sizes, fmt, where, res, stats, C.byref(done))
        if status != capi.LL_OK:
            raise SequenceError(status, self.ctx._lib.ll_last_error(self.ctx.h).decode(), done.value, [(res[i], stats[i]) for i in range(done.value)])
        return [(res[i], stats[i]) for i in range(k)]

    def pose(self):
        q, t, f = np.empty(4), np.empty(3), C.c_int()
        self.ctx.check(self.ctx._lib.ll_mapper_pose(self.h, q.ctypes.data, t.ctypes.data, C.byref(f)))
        return q, t, f.value

    def whole_map(self) -> Map:
        """A new Map of the mapper's whole map (ll_mapper_whole_map): matching mode 0, the VoxelGrid of the live history window (what the next
        refresh indexes); mode 1, the VoxelGrid of every live point of the cell maps.  The mapper is not modified."""
        h = C.c_void_p()
        self.ctx.check(self.ctx._lib.ll_mapper_whole_map(self.h, C.byref(h)))
        m = Map.__new__(Map)
        m.ctx, m.h = self.ctx, h
        return m

    def set_pose(self, q_wxyz, t):
        """The pose the next step seeds from (ll_mapper_set_pose): e.g. a relocalized pose after a load or a tracking loss."""
        q = np.ascontiguousarray(q_wxyz, np.float64)
        tt = np.ascontiguousarray(t, np.float64)
        self.ctx.check(self.ctx._lib.ll_mapper_set_pose(self.h, q.ctypes.data, tt.ctypes.data))

    def set_recovery(self, enable: bool = True, **kw):
        """Tracking-loss recovery (ll_mapper_set_recovery; DESIGN.md §4.3.2): from now on a bad step (rejected, or inlier_threshold above
        max_inlier_threshold) is held back, and after lost_after of them in a row every bad step relocalizes the step's features in the mapper's
        own map.  kw overrides fields of ll_mapper_recovery_default; enable=False turns recovery off.  Returns the capi.RecoveryCfg in force."""
        if not enable:
            self.ctx.check(self.ctx._lib.ll_mapper_set_recovery(self.h, None))
            return None
        cfg = capi.RecoveryCfg()
        self.ctx._lib.ll_mapper_recovery_default(C.byref(cfg))
        for k, v in kw.items():
            if not hasattr(cfg, k):
                raise AttributeError(k)
            setattr(cfg, k, v)
        self.ctx.check(self.ctx._lib.ll_mapper_set_recovery(self.h, C.byref(cfg)))
        return cfg

    def recovery_log(self):
        """The recovery log entries since the last read (capi.RecoveryStep, oldest first) and how many were overwritten unread."""
        out, total = [], 0
        buf, n, dropped = (capi.RecoveryStep * capi.LL_RECOVERY_LOG)(), C.c_int(), C.c_int()
        while True:
            self.ctx.check(self.ctx._lib.ll_mapper_recovery_read(self.h, buf, capi.LL_RECOVERY_LOG, C.byref(n), C.byref(dropped)))
            total += dropped.value
            out += [capi.RecoveryStep.from_buffer_copy(buf[i]) for i in range(n.value)]
            if n.value < capi.LL_RECOVERY_LOG:
                return out, total

    def set_loop_closure(self, enable: bool = True, **kw):
        """Loop closure (ll_mapper_set_loop_closure; DESIGN.md §4.6): from now on every appended step feeds the keyframes of the full-resolution map,
        and each closed keyframe is searched against the earlier ones until the first loop closes (set_loop_policy: further loops).  kw overrides fields of
        ll_mapper_loop_closure_default (loop=dict(...) the search's gates); enable=False turns it off.  Returns the capi.LoopClosureCfg in force."""
        if not enable:
            self.ctx.check(self.ctx._lib.ll_mapper_set_loop_closure(self.h, None))
            return None
        cfg = capi.LoopClosureCfg()
        self.ctx._lib.ll_mapper_loop_closure_default(C.byref(cfg))
        for k, v in kw.items():
            if not hasattr(cfg, k):
                raise AttributeError(k)
            if k == "loop" and isinstance(v, dict):
                for kk, vv in v.items():
                    if not hasattr(cfg.loop, kk):
                        raise AttributeError(kk)
                    setattr(cfg.loop, kk, vv)
            else:
                setattr(cfg, k, v)
        self.ctx.check(self.ctx._lib.ll_mapper_set_loop_closure(self.h, C.byref(cfg)))
        return cfg

    def set_loop_policy(self, max_loops: int = 1, min_keyframes_between_loops: int = 0):
        """Loops after the first (ll_mapper_set_loop_policy): close up to max_loops loops, the newest keyframes of two loops at least
        min_keyframes_between_loops apart; every loop edge joins one pose graph.  The defaults are the reference's (first loop, then stop).  Set
        after set_loop_closure (which resets it) and before the first loop; a refused policy raises and changes nothing.  Returns the
        capi.LoopPolicy in force."""
        p = capi.LoopPolicy(max_loops=max_loops, min_keyframes_between_loops=min_keyframes_between_loops)
        self.ctx.check(self.ctx._lib.ll_mapper_set_loop_policy(self.h, C.byref(p)))
        return p

    def set_loop_feedback(self, on: bool = True):
        """Loop feedback (ll_mapper_set_loop_feedback; matching mode 0): after each loop the history windows and the pose move onto the
        optimized trajectory, and loop closure goes on in the odometry frame.  Set after set_loop_closure (which turns it off) and before the
        first loop; a refusal raises and changes nothing."""
        self.ctx.check(self.ctx._lib.ll_mapper_set_loop_feedback(self.h, int(bool(on))))

    def loop_correction(self):
        """(q wxyz, t, n_applied) (ll_mapper_loop_correction_read): the correction applied last and how many were applied."""
        q, t, n = np.zeros(4), np.zeros(3), C.c_int()
        self.ctx.check(self.ctx._lib.ll_mapper_loop_correction_read(self.h, q.ctypes.data, t.ctypes.data, C.byref(n)))
        return q, t, n.value

    def loop_edges(self):
        """Every loop edge so far, in closing order (ll_mapper_loop_edges): a list of capi.PgEdge."""
        n = C.c_int()
        self.ctx.check(self.ctx._lib.ll_mapper_loop_edges(self.h, None, 0, C.byref(n)))
        buf = (capi.PgEdge * max(n.value, 1))()
        self.ctx.check(self.ctx._lib.ll_mapper_loop_edges(self.h, buf, n.value, C.byref(n)))
        return [capi.PgEdge.from_buffer_copy(buf[i]) for i in range(n.value)]

    def loop_log(self):
        """The loop-closure events since the last read (capi.LoopEvent, oldest first) and how many were overwritten unread."""
        out, total = [], 0
        buf, n, dropped = (capi.LoopEvent * capi.LL_LOOP_LOG)(), C.c_int(), C.c_int()
        while True:
            self.ctx.check(self.ctx._lib.ll_mapper_loop_read(self.h, buf, capi.LL_LOOP_LOG, C.byref(n), C.byref(dropped)))
            total += dropped.value
            out += [capi.LoopEvent.from_buffer_copy(buf[i]) for i in range(n.value)]
            if n.value < capi.LL_LOOP_LOG:
                return out, total

    def loop_result(self):
        """{"closed": bool, "poses_ori", "poses_opt": float64 [n, 7] (q w, x, y, z, t), "edge": capi.PgEdge} (ll_mapper_loop_result): poses_opt is the
        latest optimization's for the keyframes it covered and poses_ori after them; edge the latest loop edge."""
        L = self.ctx._lib
        n, closed = C.c_int(), C.c_int()
        self.ctx.check(L.ll_mapper_loop_result(self.h, C.byref(n), C.byref(closed), None, None, 0, None))
        ori, opt, edge = (capi.Pose * max(n.value, 1))(), (capi.Pose * max(n.value, 1))(), capi.PgEdge()
        self.ctx.check(L.ll_mapper_loop_result(self.h, C.byref(n), C.byref(closed), ori, opt, n.value, C.byref(edge)))
        as_np = lambda P: np.array([list(P[i].q_wxyz) + list(P[i].t) for i in range(n.value)], np.float64).reshape(n.value, 7)
        return {"closed": bool(closed.value), "poses_ori": as_np(ori), "poses_opt": as_np(opt), "edge": edge}

    def loop_cloud(self, k: int):
        """The refined cloud of published keyframe k of the latest loop (ll_mapper_loop_cloud), float32 [n, 4]."""
        n = C.c_size_t()
        self.ctx.check(self.ctx._lib.ll_mapper_loop_cloud(self.h, int(k), None, 0, C.byref(n), None))
        out = np.zeros((n.value, 4), np.float32)
        if n.value:
            self.ctx.check(self.ctx._lib.ll_mapper_loop_cloud(self.h, int(k), out.ctypes.data, n.value, C.byref(n), None))
        return out

    def save_loop(self) -> bytes:
        """The loop closure as a loop image of its own (ll_mapper_loop_save; format in include/loamlivox_b200.h).  Save it with save() at the
        same step; load() of the mapper image then load_loop() of this one continue bit for bit as this mapper does.  Raises when loop closure
        is off.  The mapper is not modified (its event log is not drained)."""
        n = C.c_size_t()
        self.ctx.check(self.ctx._lib.ll_mapper_loop_save(self.h, None, 0, C.byref(n)))
        buf = bytearray(n.value)
        self.ctx.check(self.ctx._lib.ll_mapper_loop_save(self.h, (C.c_char * len(buf)).from_buffer(buf), len(buf), C.byref(n)))
        return bytes(buf)

    def load_loop(self, image, **alloc):
        """Restore loop closure from a loop image onto this mapper (ll_mapper_loop_load), replacing any it has.  alloc may set max_cells,
        reserve_map_points, reserve_history_points and reserve_keyframes, which size the allocations; everything else is the image's config.
        A refused image raises and changes nothing."""
        img = np.frombuffer(image, np.uint8)
        cfg = None
        if alloc:
            loop_image_info(image)   # validated before its config is read
            off = int(np.frombuffer(image, np.uint64, count=1, offset=24 + 16 * capi.LL_LOOP_IMAGE_CONFIG)[0])
            cfg = capi.LoopClosureCfg.from_buffer_copy(bytes(image[off:off + C.sizeof(capi.LoopClosureCfg)]))
            for k, v in alloc.items():
                if k not in ("max_cells", "reserve_map_points", "reserve_history_points", "reserve_keyframes"):
                    raise AttributeError(f"{k}: only the allocation sizes can differ from the image's config")
                setattr(cfg, k, v)
        self.ctx.check(self.ctx._lib.ll_mapper_loop_load(self.h, img.ctypes.data, img.shape[0], C.byref(cfg) if cfg is not None else None))

    def recovery_last_inputs(self):
        """What the last relocalization attempt passed to the search (ll_mapper_recovery_last_inputs): {"corner", "surf", "score_corner",
        "score_surf": float32 [n, 4]; "rot_coarse", "rot_fine": [n, 4]; "coarse": RelocCfg; "fine": RelocFineCfg; "tmpl": RegState}; the cfgs point
        at the returned rotation arrays."""
        L = self.ctx._lib
        n = (C.c_size_t * 4)()
        coarse, fine, tmpl = capi.RelocCfg(), capi.RelocFineCfg(), capi.RegState()
        self.ctx.check(L.ll_mapper_recovery_last_inputs(self.h, C.byref(coarse), C.byref(fine), C.byref(tmpl), n, None, None, None, None, 0, None, None, 0))
        cap = max(max(n), 1)
        pts = [np.zeros((cap, 4), np.float32) for _ in range(4)]
        nrot = max(coarse.n_rot, fine.n_rot)
        rc, rf = np.zeros((nrot, 4)), np.zeros((nrot, 4))
        self.ctx.check(L.ll_mapper_recovery_last_inputs(self.h, C.byref(coarse), C.byref(fine), C.byref(tmpl), n, *[p.ctypes.data for p in pts], cap,
                                                        rc.ctypes.data, rf.ctypes.data, nrot))
        rc, rf = np.ascontiguousarray(rc[:coarse.n_rot]), np.ascontiguousarray(rf[:fine.n_rot])
        coarse.rot_wxyz = rc.ctypes.data_as(C.POINTER(C.c_double))
        fine.rot_wxyz = rf.ctypes.data_as(C.POINTER(C.c_double))
        names = ("corner", "surf", "score_corner", "score_surf")
        out = {k: pts[i][:n[i]].copy() for i, k in enumerate(names)}
        out.update(rot_coarse=rc, rot_fine=rf, coarse=coarse, fine=fine, tmpl=tmpl)
        return out

    def save(self) -> bytes:
        """The whole mapper as one byte image (ll_mapper_save; the format is specified in include/loamlivox_b200.h): Laser_mapping.load of
        it, on any context, continues bit for bit as this mapper does.  The mapper is not modified."""
        n = C.c_size_t()
        self.ctx.check(self.ctx._lib.ll_mapper_save(self.h, None, 0, C.byref(n)))
        buf = bytearray(n.value)
        self.ctx.check(self.ctx._lib.ll_mapper_save(self.h, (C.c_char * len(buf)).from_buffer(buf), len(buf), C.byref(n)))
        return bytes(buf)

    @classmethod
    def load(cls, ctx: Context, image, **alloc) -> "Laser_mapping":
        """A mapper on ctx in the state of `image` (ll_mapper_load).  alloc may set max_cells, reserve_map_points and reserve_store_points,
        which size the new mapper's buffers; everything else is the image's config.  A refused image raises and creates nothing."""
        img = np.frombuffer(image, np.uint8)
        cfg = None
        if alloc:
            image_info(image)   # validated before its config is read
            cfg = image_config(image)
            for k, v in alloc.items():
                if k not in ("max_cells", "reserve_map_points", "reserve_store_points"):
                    raise AttributeError(f"{k}: only the buffer sizes can differ from the image's config")
                setattr(cfg, k, v)
        h = C.c_void_p()
        ctx.check(ctx._lib.ll_mapper_load(ctx.h, img.ctypes.data, img.shape[0], C.byref(cfg) if cfg is not None else None, C.byref(h)))
        self = cls.__new__(cls)
        self.ctx, self.h = ctx, h
        self.cfg = image_config(image)   # what the mapper saves; alloc only sized its buffers
        return self


def image_config(image) -> capi.MapperConfig:
    """The ll_mapper_config recorded in a mapper image (section LL_IMAGE_CONFIG; the image is not validated here)."""
    off = int(np.frombuffer(image, np.uint64, count=1, offset=24 + 16 * capi.LL_IMAGE_CONFIG)[0])
    return capi.MapperConfig.from_buffer_copy(bytes(image[off:off + C.sizeof(capi.MapperConfig)]))


def image_info(image) -> dict:
    """Validate a mapper image completely on the host (no context, no GPU) and report what is in it (ll_mapper_image_info): per class
    ([corner, surface]) the history window's segments and points, the snapshot's points, the cell maps' cells, live points and frame index."""
    img = np.frombuffer(image, np.uint8)
    info = capi.ImageInfo()
    st = capi.lib().ll_mapper_image_info(img.ctypes.data, img.shape[0], C.byref(info))
    if st != capi.LL_OK:
        raise LoamLivoxError(f"status {st}: mapper image refused")
    return {n: (list(getattr(info, n)) if isinstance(getattr(info, n), C.Array) else getattr(info, n)) for n, _ in capi.ImageInfo._fields_ if n != "reserved"}


def loop_correction(poses_ori, poses_opt, f, s: int):
    """ll_loop_correction (host only): the correction (q wxyz, t) of the step with frame index s, for keyframes closed at frame indices f
    (strictly ascending) with poses_ori / poses_opt [n, 7] (q w, x, y, z, t)."""
    ori, opt = (np.ascontiguousarray(np.asarray(P, np.float64).reshape(-1, 7)) for P in (poses_ori, poses_opt))
    fa = np.ascontiguousarray(np.asarray(f, np.int32))
    n = fa.shape[0]
    if ori.shape[0] != n or opt.shape[0] != n:
        raise ValueError("poses_ori, poses_opt and f must have one entry per keyframe")
    q, t = np.zeros(4), np.zeros(3)
    st = capi.lib().ll_loop_correction(ori.ctypes.data_as(C.POINTER(capi.Pose)), opt.ctypes.data_as(C.POINTER(capi.Pose)), fa.ctypes.data, n, int(s),
                                       q.ctypes.data, t.ctypes.data)
    if st != capi.LL_OK:
        raise LoamLivoxError(f"status {st}: ll_loop_correction refused its inputs")
    return q, t


def loop_image_info(image) -> dict:
    """Validate a loop image completely on the host (no context, no GPU) and report what is in it (ll_loop_image_info)."""
    img = np.frombuffer(image, np.uint8) if len(image) else np.zeros(1, np.uint8)
    info = capi.LoopImageSummary()
    st = capi.lib().ll_loop_image_info(img.ctypes.data, len(image), C.byref(info))
    if st != capi.LL_OK:
        raise LoamLivoxError(f"status {st}: loop image refused")
    return {n: getattr(info, n) for n, _ in capi.LoopImageSummary._fields_}


class Laser_feature:
    """The Velodyne branch of Laser_feature::laserCloudHandler (loam_livox/source/laser_feature_extractor.hpp:393-825; scan_line 16 or 64)
    on the device.  laserCloudHandler(cloud) returns the five clouds the reference publishes: /laser_points_2, /laser_cloud_sharp,
    /laser_cloud_less_sharp, /laser_cloud_flat, /laser_cloud_less_flat.  The 20-frame start-up delay stays the caller's."""

    CLOUDS = ("full", "sharp", "less_sharp", "flat", "less_flat")

    def __init__(self, ctx: Context, scan_line: int = 16, minimum_range: float = 0.1, plane_resolution: float = 0.4, max_points: int = 400000):
        self.ctx = ctx
        cfg = capi.default_spin_cfg(scan_line=scan_line, minimum_range=minimum_range, plane_resolution=plane_resolution, max_points=max_points)
        h = C.c_void_p()
        ctx.check(ctx._lib.ll_spin_create(ctx.h, C.byref(cfg), C.byref(h)))
        self.h = h
        self.counts = np.zeros(5, np.uint64)

    def close(self):
        if getattr(self, "h", None):
            self.ctx._lib.ll_spin_release(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def extract(self, raw, where=capi.LL_HOST, n=None, fmt=None):
        """One cloud: a float32 array [n, 4] / [n, 8] (where = LL_HOST), or a device pointer with n and fmt (LL_DEVICE); returns the counts."""
        counts = (C.c_size_t * 5)()
        if where == capi.LL_HOST and fmt is None:
            raw, fmt = _pts(raw)
            ptr, n = raw.ctypes.data, raw.shape[0]
        elif where == capi.LL_HOST:
            ptr = raw.ctypes.data if isinstance(raw, np.ndarray) else C.cast(C.c_char_p(raw), C.c_void_p).value
        else:
            ptr = raw
        self.ctx.check(self.ctx._lib.ll_spin_extract(self.h, ptr, n, fmt, where, counts))
        self.counts = np.array(list(counts), np.uint64)
        return self.counts

    def extract_from_pointcloud2(self, data: bytes, n_points: int):
        """A sensor_msgs/PointCloud2 payload in the context's point layout (Context.set_point_layout)."""
        buf = np.frombuffer(data, np.uint8)
        return self.extract(np.ascontiguousarray(buf), capi.LL_HOST, n_points, capi.LL_FMT_STRIDED)

    def cloud(self, which: int):
        n, dev = C.c_size_t(), C.c_void_p()
        self.ctx.check(self.ctx._lib.ll_spin_cloud(self.h, which, None, 0, C.byref(n), C.byref(dev)))
        out = np.zeros((n.value, 4), np.float32)
        self.ctx.check(self.ctx._lib.ll_spin_cloud(self.h, which, out.ctypes.data, n.value, C.byref(n), None))
        return out

    def device_cloud(self, which: int):
        """(device pointer, point count) of a cloud, valid until the next extract: an LL_DEVICE input of ll_register / ll_map_build."""
        n, dev = C.c_size_t(), C.c_void_p()
        self.ctx.check(self.ctx._lib.ll_spin_cloud(self.h, which, None, 0, C.byref(n), C.byref(dev)))
        return dev.value, n.value

    def laserCloudHandler(self, raw):
        self.extract(raw)
        return {name: self.cloud(k) for k, name in enumerate(self.CLOUDS)}

    def point_info(self):
        """(ring, curvature, picked before the selection, label) per point of the full cloud."""
        n = C.c_size_t()
        self.ctx.check(self.ctx._lib.ll_spin_point_info(self.h, None, None, None, None, 0, C.byref(n)))
        k = n.value
        ring, curv, picked, label = np.zeros(k, np.int32), np.zeros(k, np.float32), np.zeros(k, np.int32), np.zeros(k, np.int32)
        self.ctx.check(self.ctx._lib.ll_spin_point_info(self.h, ring.ctypes.data, curv.ctypes.data, picked.ctypes.data, label.ctypes.data, k, C.byref(n)))
        return ring, curv, picked, label

    def chains(self):
        """(number of independent chains of the last selection, longest chain in points)."""
        a, b = C.c_int(), C.c_int()
        self.ctx.check(self.ctx._lib.ll_spin_chains(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value
