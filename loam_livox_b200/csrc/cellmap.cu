// Device-resident voxel-cell map (a14) as the matching path uses it in matching_mode 1.
//
// Replaces, on the reference side:
//   Points_cloud_map<float>::append_cloud / set_point_cloud / find_cell / add_cell / find_cell_center
//                                              loam_livox/source/cell_map_keyframe.hpp:556-571,578-672,681-758
//   Points_cloud_cell::append_pt / get_pointcloud / set_pointcloud        :331-351,378-419   (cells keep xyz only)
//   find_cells_in_radius + if_pt_in_fov + per-cell VoxelGrid + down-sample-and-replace (update_buff_for_matching, mode 1)
//                                              loam_livox/source/laser_mapping.hpp:310-324,471-516, cell_map_keyframe.hpp:761-788
//
// Layout: an open-addressing hash table of cells keyed by the packed integer cell index (k, j, i) (21 bits each, so that ascending key ==
// ascending (k, j, i), the order in which the cells are visited), with per-cell frame stamps and an epoch; and ONE flat point store
// (float4 xyz, cell slot, epoch).  A point is alive iff its epoch equals its cell's epoch: the reference's "revisit" (a cell untouched
// for >= threshold frames is replaced by an empty one) is a single epoch increment.  Down-sample-and-replace rebuilds the store by
// compaction.  Everything stays in HBM; the host only mirrors three counters.
// Compiled with -fmad=false (cell indices, voxel indices and centroids must round like the scalar CPU code).
#include <cub/cub.cuh>
#include <cmath>
#include "common.cuh"
#include "kernels.cuh"
#include "exact_math.cuh"
#include "cellmap.cuh"

#define CM_MAX_VOXELS_PER_CELL 512.0  // finest leaf an assembly accepts: cell size / 512 (see ll_cellmap_assemble)
#define CM_VOXEL_BIAS 1024            // a cell's points lie within one cell of its lower corner: 512 voxels and this margin fit 13 bits

__device__ __forceinline__ unsigned cm_hash(unsigned long long key, unsigned mask) { return (unsigned)((key * 0x9E3779B97F4A7C15ull) >> 32) & mask; }

// pass 1: cell lookup / creation for every new point (find_cell with if_add = 1)
__global__ void cm_locate_kernel(const float4* __restrict__ in, int n, float box, float half, int cur, unsigned long long* keys, unsigned mask, int* create_frame, int* last_update,
                                 int* epoch, int* bump, int* counters, int* __restrict__ slot_out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const float4 p = in[t];
  if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) { slot_out[t] = -1; return; }
  const float fi = roundf((p.x - half) / box), fj = roundf((p.y - half) / box), fk = roundf((p.z - half) / box);
  const float lo = -(float)CM_BIAS, hi = (float)(CM_BIAS - 1);
  if (!(fi >= lo && fi <= hi && fj >= lo && fj <= hi && fk >= lo && fk <= hi)) { slot_out[t] = -1; atomicAdd(&counters[2], 1); return; }
  const int i = (int)fi, j = (int)fj, k = (int)fk;
  const unsigned long long key = cm_pack(k, j, i);
  unsigned h = cm_hash(key, mask);
  for (;;) {
    const unsigned long long prev = atomicCAS(&keys[h], CM_EMPTY, key);
    if (prev == CM_EMPTY) { create_frame[h] = cur; last_update[h] = cur; epoch[h] = 0; bump[h] = -1; atomicAdd(&counters[0], 1); break; }
    if (prev == key) break;
    h = (h + 1) & mask;
  }
  slot_out[t] = (int)h;
}
// pass 2: revisit handling (find_cell with if_treat_revisit = 1): one epoch bump per stale cell and call
__global__ void cm_revisit_kernel(const int* __restrict__ slot_in, int n, int cur, int threshold, const int* __restrict__ create_frame, const int* __restrict__ last_update, int* epoch, int* bump) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const int s = slot_in[t]; if (s < 0) return;
  if (create_frame[s] != cur && (cur - last_update[s]) >= threshold) { if (atomicExch(&bump[s], cur) != cur) atomicAdd(&epoch[s], 1); }
}
// pass 3: append the points (append_pt) and stamp the cells
__global__ void cm_store_kernel(const float4* __restrict__ in, const int* __restrict__ slot_in, int n, int cur, int base, const int* __restrict__ epoch, const int* __restrict__ bump,
                                int* create_frame, int* last_update, float4* pts, int* pt_slot, int* pt_epoch) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const int s = slot_in[t]; const float4 p = in[t];
  pts[base + t] = make_float4(p.x, p.y, p.z, 0.f);
  pt_slot[base + t] = s; pt_epoch[base + t] = s >= 0 ? epoch[s] : -1;
  if (s >= 0) { last_update[s] = cur; if (bump[s] == cur) create_frame[s] = cur; }
}

// ---- assemble -----------------------------------------------------------------------------------------------------------------
struct CmView { double q[4]; double t[3]; float sp[3]; double r2; float fov; float box, half; };

__global__ void cm_select_cells_kernel(const unsigned long long* __restrict__ keys, int cap, CmView v, unsigned char* __restrict__ sel) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= cap) return;
  const unsigned long long key = keys[s];
  unsigned char f = 0;
  if (key != CM_EMPTY) {
    int k, j, i; cm_unpack(key, k, j, i);
    const float cx = (float)i * v.box + v.half, cy = (float)j * v.box + v.half, cz = (float)k * v.box + v.half;
    const float dx = cx - v.sp[0], dy = cy - v.sp[1], dz = cz - v.sp[2];
    if ((double)(dx * dx + (dy * dy + dz * dz)) <= v.r2) {   // octree radiusSearch: float squaredNorm (Eigen order) <= double radius^2
      // if_pt_in_fov: pt_affine = q_w_curr.inverse() * (centre - t_w_curr); x >= 0 and acos(|x| / |pt_affine|) * 57.3 < maximum_in_fov_angle
      const double n2 = v.q[0] * v.q[0] + v.q[1] * v.q[1] + v.q[2] * v.q[2] + v.q[3] * v.q[3];
      const double qi[4] = {v.q[0] / n2, -v.q[1] / n2, -v.q[2] / n2, -v.q[3] / n2};
      double ax, ay, az; qrot_d(qi, (double)cx - v.t[0], (double)cy - v.t[1], (double)cz - v.t[2], ax, ay, az);
      if (!(ax < 0)) {
        const double an = sqrt(ax * ax + (ay * ay + az * az));
        float angle = 0.0f;
        if (an != 0.0) angle = (float)acos(fabs(ax * 1.0 + (ay * 0.0 + az * 0.0)) / (an * 1.0));
        if ((double)angle * 57.3 < (double)v.fov) f = 1;
      }
    }
  }
  sel[s] = f;
}
__global__ void cm_rank_kernel(const int* __restrict__ sorted_slots, int n_sel, int* __restrict__ rank_of_slot) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n_sel) rank_of_slot[sorted_slots[r]] = r;
}
__global__ void cm_gather_keys_kernel(const unsigned long long* __restrict__ keys, const int* __restrict__ slots, const int* __restrict__ d_n, unsigned long long* __restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < *d_n) out[r] = keys[slots[r]];
}
// flags per stored point: 1 = alive and in a selected cell, 2 = alive and not selected (kept as is), 0 = dead
__global__ void cm_point_flags_kernel(const int* __restrict__ pt_slot, const int* __restrict__ pt_epoch, int n, const int* __restrict__ epoch, const unsigned char* __restrict__ sel,
                                      unsigned char* __restrict__ f_sel, unsigned char* __restrict__ f_keep) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const int s = pt_slot[t];
  const bool alive = s >= 0 && pt_epoch[t] == epoch[s];
  f_sel[t] = (alive && sel[s]) ? 1 : 0; f_keep[t] = (alive && !sel[s]) ? 1 : 0;
}
__global__ void cm_count_alive_kernel(const int* __restrict__ pt_slot, const int* __restrict__ pt_epoch, int n, const int* __restrict__ epoch, int* out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const bool alive = t < n && pt_slot[t] >= 0 && pt_epoch[t] == epoch[pt_slot[t]];
  const unsigned b = __ballot_sync(0xffffffffu, alive);
  if ((threadIdx.x & 31) == 0 && b) atomicAdd(out, __popc(b));
}
// sort key of a selected point: (rank of its cell, voxel z, y, x) with voxel = floor(p / leaf) relative to a per-cell origin
__global__ void cm_voxel_keys_kernel(const float4* __restrict__ pts, const int* __restrict__ pt_slot, const int* __restrict__ idx, const int* __restrict__ d_n, const unsigned long long* __restrict__ keys,
                                     const int* __restrict__ rank_of_slot, float box, float half, float inv, unsigned long long* __restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= *d_n) return;
  const int t = idx[r]; const int s = pt_slot[t]; const float4 p = pts[t];
  int k, j, i; cm_unpack(keys[s], k, j, i);
  const float ox = (float)i * box, oy = (float)j * box, oz = (float)k * box;   // lower corner of the cell (centre - half)
  const int bx = (int)floorf(ox * inv) - CM_VOXEL_BIAS, by = (int)floorf(oy * inv) - CM_VOXEL_BIAS, bz = (int)floorf(oz * inv) - CM_VOXEL_BIAS;
  const int vx = (int)floorf(p.x * inv) - bx, vy = (int)floorf(p.y * inv) - by, vz = (int)floorf(p.z * inv) - bz;
  out[r] = ((unsigned long long)rank_of_slot[s] << 39) | ((unsigned long long)(vz & 0x1fff) << 26) | ((unsigned long long)(vy & 0x1fff) << 13) | (unsigned long long)(vx & 0x1fff);
}
__global__ void cm_heads_kernel(const unsigned long long* __restrict__ k, const int* __restrict__ d_n, unsigned char* __restrict__ flags, int cap) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= cap) return;
  flags[r] = (r < *d_n && (r == 0 || k[r] != k[r - 1])) ? 1 : 0;
}
// one thread per (cell, voxel): float sums in stored order (CentroidPoint<PointXYZI>; intensity is 0)
__global__ void cm_centroid_kernel(const float4* __restrict__ pts, const int* __restrict__ pt_slot, const int* __restrict__ sorted_idx, const int* __restrict__ seg, const int* __restrict__ d_nseg,
                                   const int* __restrict__ d_nsel, float4* __restrict__ out, int* __restrict__ out_slot) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  const int nseg = *d_nseg;
  if (s >= nseg) return;
  const int b = seg[s], e = (s + 1 < nseg) ? seg[s + 1] : *d_nsel;
  float sx = 0.f, sy = 0.f, sz = 0.f, si = 0.f;
  for (int r = b; r < e; r++) { const float4 p = pts[sorted_idx[r]]; sx += p.x; sy += p.y; sz += p.z; si += 0.f; }
  const float c = (float)(e - b);
  out[s] = make_float4(sx / c, sy / c, sz / c, si / c);
  out_slot[s] = pt_slot[sorted_idx[b]];
}
// rebuild of the point store: kept points (compacted, order preserved) followed by the centroids of the down-sampled cells
__global__ void cm_rebuild_kernel(const float4* __restrict__ pts, const int* __restrict__ pt_slot, const int* __restrict__ pt_epoch, const int* __restrict__ keep_idx, const int* __restrict__ d_nkeep,
                                  const float4* __restrict__ cen, const int* __restrict__ cen_slot, const int* __restrict__ d_ncen, const int* __restrict__ epoch,
                                  float4* __restrict__ npts, int* __restrict__ nslot, int* __restrict__ nepoch, int cap) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int nk = *d_nkeep, nc = *d_ncen;
  if (t < nk) { const int o = keep_idx[t]; npts[t] = pts[o]; nslot[t] = pt_slot[o]; nepoch[t] = pt_epoch[o]; }
  else if (t < nk + nc && t < cap) { const int c = t - nk; const float4 p = cen[c]; npts[t] = make_float4(p.x, p.y, p.z, 0.f); nslot[t] = cen_slot[c]; nepoch[t] = epoch[cen_slot[c]]; }
}

// A point store of `cap` points: points | their cells | the cells' epochs when stored
struct CmStore {
  float4* pts; int* slot; int* epoch;
  void layout(Carve& c, size_t cap) { pts = c.take<float4>(cap); slot = c.take<int>(cap); epoch = c.take<int>(cap); }
};
static inline size_t cm_store_bytes(size_t cap) { CmStore st; return layout_bytes([&](Carve& c) { st.layout(c, cap); }); }
// Store capacity for `need` points, growing from `cur` (0: none yet) by doubling
static inline size_t cm_store_cap(size_t cur, size_t need) { size_t cap = cur > 0 ? cur : (1 << 16); while (cap < need) cap *= 2; return cap; }
static const size_t CM_MAX_STORE = (size_t)1 << 30;
// An append's upload of n points and their cell slots
struct CmAppend {
  float4* in; int* slot;
  void layout(Carve& c, size_t n) { in = c.take<float4>(n); slot = c.take<int>(n); }
};

static int cm_reserve_store(ll_ctx* ctx, ll_cellmap* m, int need) {
  if (need <= m->cap_pts) return LL_OK;
  const int cap = (int)cm_store_cap((size_t)m->cap_pts, (size_t)need);
  CmStore st;
  if (m->n_pts == 0 && m->store_buf.cap >= cm_store_bytes((size_t)cap)) {   // nothing to carry over and the (pre-reserved) allocation is large enough
    LL_CUDA(ctx, m->store_buf.carve([&](Carve& c) { st.layout(c, cap); }));
    m->pts = st.pts; m->pt_slot = st.slot; m->pt_epoch = st.epoch;
    m->cap_pts = cap; return LL_OK;
  }
  DevBuf nb; LL_CUDA(ctx, nb.carve([&](Carve& c) { st.layout(c, cap); }));
  float4* np = st.pts; int* ns = st.slot; int* ne = st.epoch;
  if (m->n_pts > 0) {
    LL_CUDA(ctx, cudaMemcpyAsync(np, m->pts, (size_t)m->n_pts * 16, cudaMemcpyDeviceToDevice, ctx->stream));
    LL_CUDA(ctx, cudaMemcpyAsync(ns, m->pt_slot, (size_t)m->n_pts * 4, cudaMemcpyDeviceToDevice, ctx->stream));
    LL_CUDA(ctx, cudaMemcpyAsync(ne, m->pt_epoch, (size_t)m->n_pts * 4, cudaMemcpyDeviceToDevice, ctx->stream));
    LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  m->store_buf.release(); m->store_buf = nb; m->pts = np; m->pt_slot = ns; m->pt_epoch = ne; m->cap_pts = cap;
  return LL_OK;
}

// The assembly's scratch over a table of T slots and a store of N points
struct CmAssemble {
  size_t cub_bytes = 0;   // CUB temporaries: select over the table / the store, 64-bit pair sort of the selected points
  unsigned char* sel; int* cslots; unsigned long long* ckeys; unsigned long long* ckeys2; int* cslots2; int* rank;
  unsigned char* fsel; unsigned char* fkeep; int* isel; int* ikeep; unsigned long long* vk; unsigned long long* vk2; int* isel2;
  unsigned char* heads; int* seg; int* cslot; int* cnt; char* cub_tmp;
  CmAssemble(int T, int N) {
    const int big = T > N ? T : N;
    size_t cub_a = 0, cub_b = 0;
    cub::DeviceSelect::Flagged(nullptr, cub_a, cub::CountingInputIterator<int>(0), (unsigned char*)nullptr, (int*)nullptr, (int*)nullptr, big);
    cub::DeviceRadixSort::SortPairs(nullptr, cub_b, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int*)nullptr, (int*)nullptr, big, 0, 64);
    cub_bytes = cub_a > cub_b ? cub_a : cub_b;
  }
  void layout(Carve& c, size_t T, size_t N) {
    sel = c.take<unsigned char>(T); cslots = c.take<int>(T); ckeys = c.take<unsigned long long>(T); ckeys2 = c.take<unsigned long long>(T); cslots2 = c.take<int>(T); rank = c.take<int>(T);
    fsel = c.take<unsigned char>(N); fkeep = c.take<unsigned char>(N); isel = c.take<int>(N); ikeep = c.take<int>(N); vk = c.take<unsigned long long>(N); vk2 = c.take<unsigned long long>(N);
    isel2 = c.take<int>(N); heads = c.take<unsigned char>(N); seg = c.take<int>(N); cslot = c.take<int>(N);
    cnt = c.take<int>(16); cub_tmp = c.take<char>(cub_bytes);
  }
};
static size_t cm_assemble_bytes(int T, int N) { CmAssemble a(T, N); return layout_bytes([&](Carve& c) { a.layout(c, T, N); }); }

int64_t table_capacity(int max_cells) { int64_t cap = 1 << 12; const int64_t want = 2 * (int64_t)(max_cells > 0 ? max_cells : (1 << 20)); while (cap < want) cap <<= 1; return cap; }

extern "C" {

// Size every buffer of the map for `store_points` stored points and appends of up to `scan_points` points, now: after this, appends and assemblies
// allocate nothing until the store outgrows the reservation (then it doubles, as before).
int ll_cellmap_reserve(ll_ctx* ctx, ll_cellmap* m, size_t store_points, size_t scan_points) {
  if (!ctx || !m) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  const size_t cap = cm_store_cap(0, store_points);
  if (cap > CM_MAX_STORE) return LL_ERR_INVALID;
  if (m->n_pts == 0) LL_CUDA(ctx, m->store_buf.reserve_floor(cm_store_bytes(cap)));
  LL_TRY(cm_reserve_store(ctx, m, (int)cap));
  LL_CUDA(ctx, m->store_alt.reserve_floor(cm_store_bytes(cap)));
  LL_CUDA(ctx, m->out_buf.reserve_floor(layout_bytes([&](Carve& c) { c.take<float4>(cap); })));
  CmAppend ap;
  if (scan_points) LL_CUDA(ctx, m->tmp_buf.reserve_floor(layout_bytes([&](Carve& c) { ap.layout(c, scan_points); })));
  LL_CUDA(ctx, ctx->scratch.reserve_floor(cm_assemble_bytes(m->table_cap, (int)cap)));
  return LL_OK;
}

int ll_cellmap_create(ll_ctx* ctx, float resolution, int revisit_threshold, int max_cells, ll_cellmap** out) {
  // revisit_threshold < 1 would replace a cell at every point that touches it (only the last point of a call would stay); it is refused
  if (!ctx || !out || !(resolution > 0.f) || revisit_threshold < 1 || max_cells > MAX_CELLS) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  ll_cellmap* m = new ll_cellmap(); m->device = ctx->device; m->resolution = resolution * 0.5f; m->revisit_threshold = revisit_threshold;
  const int cap = (int)table_capacity(max_cells);
  m->table_cap = cap;
  const cudaError_t e = m->table_buf.carve([&](Carve& c) {
    m->keys = c.take<unsigned long long>(cap);
    m->last_update = c.take<int>(cap); m->create_frame = c.take<int>(cap); m->epoch = c.take<int>(cap); m->bump = c.take<int>(cap);
    m->d_counters = c.take<int>(16);
  });
  if (e != cudaSuccess) { delete m; ctx->set_error("cell table allocation failed"); return LL_ERR_CUDA; }
  cudaMemsetAsync(m->keys, 0xff, (size_t)cap * 8, ctx->stream); cudaMemsetAsync(m->d_counters, 0, 64, ctx->stream);
  if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) { m->table_buf.release(); delete m; return LL_ERR_CUDA; }
  *out = m; return LL_OK;
}
void ll_cellmap_release(ll_cellmap* m) {
  if (!m) return;
  cudaSetDevice(m->device);
  m->table_buf.release(); m->store_buf.release(); m->store_alt.release(); m->out_buf.release(); m->tmp_buf.release(); delete m;
}
int ll_cellmap_stats(ll_ctx* ctx, ll_cellmap* m, int* cells, int* stored_points, int* frame_idx) {
  if (!ctx || !m) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  int c[2] = {0, 0};
  LL_CUDA(ctx, cudaMemsetAsync(m->d_counters + 1, 0, 4, ctx->stream));
  if (m->n_pts > 0) { cm_count_alive_kernel<<<ll_div_up(m->n_pts, 256), 256, 0, ctx->stream>>>(m->pt_slot, m->pt_epoch, m->n_pts, m->epoch, m->d_counters + 1); ctx->launches++; }
  LL_CUDA(ctx, cudaMemcpyAsync(c, m->d_counters, 8, cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  // points of replaced (revisited) cells are dead and not counted
  if (cells) *cells = c[0]; if (stored_points) *stored_points = c[1]; if (frame_idx) *frame_idx = m->current_frame_idx;
  return LL_OK;
}

// Points_cloud_map::append_cloud (cell_map_keyframe.hpp:619-672): every point goes to its 0.5 m cell; xyz only.
int ll_cellmap_append(ll_ctx* ctx, ll_cellmap* m, const void* pts, size_t n, int fmt, int where) {
  if (!ctx || !m) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  cudaStream_t s = ctx->stream;
  const bool first = m->n_cells == 0;   // append_cloud calls set_point_cloud while the map has no cell (:625-629)
  int bad = 0;
  if (n > 0) {
    LL_TRY(cm_reserve_store(ctx, m, m->n_pts + (int)n));
    CmAppend ap; LL_CUDA(ctx, m->tmp_buf.carve([&](Carve& c) { ap.layout(c, n); }));
    float4* d_in = ap.in; int* d_slot = ap.slot;
    LL_TRY(upload_cloud(ctx, s, pts, n, fmt, where, d_in));
    const float box = m->resolution * 1.0f, half = m->resolution * 0.5f;
    const int blocks = ll_div_up((int)n, 256), cur = m->current_frame_idx;
    cm_locate_kernel<<<blocks, 256, 0, s>>>(d_in, (int)n, box, half, cur, m->keys, (unsigned)(m->table_cap - 1), m->create_frame, m->last_update, m->epoch, m->bump, m->d_counters, d_slot);
    cm_revisit_kernel<<<blocks, 256, 0, s>>>(d_slot, (int)n, cur, m->revisit_threshold, m->create_frame, m->last_update, m->epoch, m->bump);
    cm_store_kernel<<<blocks, 256, 0, s>>>(d_in, d_slot, (int)n, cur, m->n_pts, m->epoch, m->bump, m->create_frame, m->last_update, m->pts, m->pt_slot, m->pt_epoch);
    ctx->launches += 3;
    LL_CUDA(ctx, cudaGetLastError());
    m->n_pts += (int)n;
    int c[3] = {0, 0, 0};
    LL_CUDA(ctx, cudaMemcpyAsync(c, m->d_counters, sizeof(c), cudaMemcpyDeviceToHost, s));
    LL_CUDA(ctx, cudaStreamSynchronize(s));
    m->n_cells = c[0];
    if (c[0] > m->table_cap / 2) { ctx->set_error("cell table more than half full: create the map with a larger max_cells"); return LL_ERR_CAPACITY; }
    if (c[2] != m->n_out_of_range) { bad = c[2] - m->n_out_of_range; m->n_out_of_range = c[2]; }
  }
  if (first) m->current_frame_idx++;   // set_point_cloud() bumps the frame index too (:616) ...
  m->current_frame_idx++;              // ... and append_cloud() always does (:666)
  if (bad) {   // the append is complete without them: they are dead slots, like non-finite points
    char msg[160]; snprintf(msg, sizeof(msg), "%d point(s) dropped: cell index beyond +-2^20 (the cell key's range)", bad);
    ctx->set_error(msg); return LL_ERR_INVALID;
  }
  return LL_OK;
}

// update_buff_for_matching, matching_mode 1, for one map (laser_mapping.hpp:475-516).  The assembled cloud stays on the device
// (*out_dev, valid until the next call on this map); it is also copied to out_host when that is not NULL (cap points).
int ll_cellmap_assemble(ll_ctx* ctx, ll_cellmap* m, const double q_wxyz[4], const double t[3], float search_range, float fov_deg, float leaf, int down_sample_replace,
                        ll_point* out_host, size_t cap, size_t* n_out, int* cells_in_fov, const ll_point** out_dev) {
  if (!ctx || !m || !q_wxyz || !t || !n_out || !(leaf > 0.f)) return LL_ERR_INVALID;
  // A leaf finer than cell / 512 is refused: PCL's per-cell VoxelGrid then depends on whether the cell's voxel count overflows int32 (it passes
  // such a cell through unfiltered), which the per-cell keys below do not reproduce.  Down to it, a cell spans at most ~700 voxels per axis.
  if ((double)m->resolution / (double)leaf > CM_MAX_VOXELS_PER_CELL) { ctx->set_error("leaf finer than cell size / 512"); return LL_ERR_INVALID; }
  cudaSetDevice(ctx->device);
  cudaStream_t s = ctx->stream;
  *n_out = 0; if (cells_in_fov) *cells_in_fov = 0; if (out_dev) *out_dev = nullptr;
  const int T = m->table_cap, N = m->n_pts;
  if (N == 0) return LL_OK;
  CmView v; for (int k = 0; k < 4; k++) v.q[k] = q_wxyz[k]; for (int k = 0; k < 3; k++) { v.t[k] = t[k]; v.sp[k] = (float)t[k]; }
  v.r2 = (double)search_range * (double)search_range; v.fov = fov_deg; v.box = m->resolution * 1.0f; v.half = m->resolution * 0.5f;
  CmAssemble a(T, N);
  LL_CUDA(ctx, ctx->scratch.carve([&](Carve& c) { a.layout(c, T, N); }));
  unsigned char* sel = a.sel; int* cslots = a.cslots; unsigned long long* ckeys = a.ckeys; unsigned long long* ckeys2 = a.ckeys2;
  int* cslots2 = a.cslots2; int* rank = a.rank; unsigned char* fsel = a.fsel; unsigned char* fkeep = a.fkeep;
  int* isel = a.isel; int* ikeep = a.ikeep; unsigned long long* vk = a.vk; unsigned long long* vk2 = a.vk2; int* isel2 = a.isel2;
  unsigned char* heads = a.heads; int* seg = a.seg; int* cslot = a.cslot; int* cnt = a.cnt; void* cub_tmp = a.cub_tmp; size_t cub_c = a.cub_bytes;
  // cnt: [0] selected cells, [1] selected points, [2] kept points, [3] segments (output points)
  float4* d_out = nullptr;
  LL_CUDA(ctx, m->out_buf.carve([&](Carve& c) { d_out = c.take<float4>(N); }));
  // 1. cells within range and inside the FOV, ranked by ascending key
  cm_select_cells_kernel<<<ll_div_up(T, 256), 256, 0, s>>>(m->keys, T, v, sel);
  LL_CUDA(ctx, cub::DeviceSelect::Flagged(cub_tmp, cub_c, cub::CountingInputIterator<int>(0), sel, cslots, cnt + 0, T, s));
  int h_cnt[4] = {0, 0, 0, 0};
  LL_CUDA(ctx, cudaMemcpyAsync(h_cnt, cnt, 4, cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  const int n_cells = h_cnt[0];
  if (cells_in_fov) *cells_in_fov = n_cells;
  if (n_cells == 0) return LL_OK;
  cm_gather_keys_kernel<<<ll_div_up(n_cells, 256), 256, 0, s>>>(m->keys, cslots, cnt + 0, ckeys);
  LL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(cub_tmp, cub_c, ckeys, ckeys2, cslots, cslots2, n_cells, 0, 64, s));
  cm_rank_kernel<<<ll_div_up(n_cells, 256), 256, 0, s>>>(cslots2, n_cells, rank);
  // 2. live points of those cells, sorted by (cell rank, voxel), stable in stored order
  cm_point_flags_kernel<<<ll_div_up(N, 256), 256, 0, s>>>(m->pt_slot, m->pt_epoch, N, m->epoch, sel, fsel, fkeep);
  LL_CUDA(ctx, cub::DeviceSelect::Flagged(cub_tmp, cub_c, cub::CountingInputIterator<int>(0), fsel, isel, cnt + 1, N, s));
  LL_CUDA(ctx, cub::DeviceSelect::Flagged(cub_tmp, cub_c, cub::CountingInputIterator<int>(0), fkeep, ikeep, cnt + 2, N, s));
  LL_CUDA(ctx, cudaMemcpyAsync(h_cnt, cnt, 12, cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  const int n_sel = h_cnt[1], n_keep = h_cnt[2];
  if (n_sel == 0) return LL_OK;
  cm_voxel_keys_kernel<<<ll_div_up(n_sel, 256), 256, 0, s>>>(m->pts, m->pt_slot, isel, cnt + 1, m->keys, rank, v.box, v.half, 1.0f / leaf, vk);
  LL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(cub_tmp, cub_c, vk, vk2, isel, isel2, n_sel, 0, 64, s));
  cm_heads_kernel<<<ll_div_up(n_sel, 256), 256, 0, s>>>(vk2, cnt + 1, heads, n_sel);
  LL_CUDA(ctx, cub::DeviceSelect::Flagged(cub_tmp, cub_c, cub::CountingInputIterator<int>(0), heads, seg, cnt + 3, n_sel, s));
  cm_centroid_kernel<<<ll_div_up(n_sel, 256), 256, 0, s>>>(m->pts, m->pt_slot, isel2, seg, cnt + 3, cnt + 1, d_out, cslot);
  LL_CUDA(ctx, cudaMemcpyAsync(h_cnt, cnt, 16, cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  const int n_cen = h_cnt[3];
  ctx->launches += 16;
  // 3. down-sample-and-replace (m_down_sample_replace = 1, laser_mapping.hpp:277,492-495,510-513): rebuild the store
  if (down_sample_replace) {
    const int n_new = n_keep + n_cen;
    const int cap_new = (int)cm_store_cap((size_t)m->cap_pts, (size_t)n_new);
    DevBuf& nb = m->store_alt;   // ping-pong: the two stores persist, so a refresh allocates nothing in steady state
    CmStore st; LL_CUDA(ctx, nb.carve([&](Carve& c) { st.layout(c, cap_new); }));
    float4* np = st.pts; int* ns = st.slot; int* ne = st.epoch;
    cm_rebuild_kernel<<<ll_div_up(n_new > 0 ? n_new : 1, 256), 256, 0, s>>>(m->pts, m->pt_slot, m->pt_epoch, ikeep, cnt + 2, d_out, cslot, cnt + 3, m->epoch, np, ns, ne, cap_new);
    { DevBuf t = m->store_buf; m->store_buf = m->store_alt; m->store_alt = t; }   // stream-ordered: later work on this stream sees the new store
    m->pts = np; m->pt_slot = ns; m->pt_epoch = ne; m->cap_pts = cap_new; m->n_pts = n_new; m->generation++;
    ctx->launches++;
  }
  *n_out = (size_t)n_cen;
  if (out_dev) *out_dev = (const ll_point*)d_out;
  if (out_host && n_cen > 0) {
    const size_t w = (size_t)n_cen < cap ? (size_t)n_cen : cap;
    LL_CUDA(ctx, cudaMemcpyAsync(out_host, d_out, w * 16, cudaMemcpyDeviceToHost, s));
    LL_CUDA(ctx, cudaStreamSynchronize(s));
  }
  LL_CUDA(ctx, cudaGetLastError());
  return LL_OK;
}

}  // extern "C"

// ---- checkpoint (ll_mapper_save / ll_mapper_load, ll_mapper_loop_save / ll_mapper_loop_load) -------------------------------------------
// A map leaves as its cells in ascending key (key, create_frame, last_update) and its live points in store order (xyz, rank of the cell in
// that list), and comes back into an empty table with every cell at epoch 0, bump -1 and every point at epoch 0.  Nothing a result depends on
// changes: the assembly ranks cells by key and keeps store order inside a voxel, and liveness is only "point epoch == cell epoch".
// With a held list (the loop image: the (slot << 32 | epoch) ids the open keyframes hold, sorted and distinct) the points of those
// incarnations leave too, and every kept point and every cell carry an incarnation ordinal (cm_ordinal); the import sets them as the epochs.
__device__ __forceinline__ bool cm_is_held(const unsigned long long* held, int n_held, int s, int e) {
  const unsigned long long id = ((unsigned long long)(unsigned)s << 32) | (unsigned)e;
  const int at = cm_lower_bound(held, n_held, id);
  return at < n_held && held[at] == id;
}
__global__ void cm_occupied_kernel(const unsigned long long* __restrict__ keys, int cap, unsigned char* __restrict__ flag) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < cap) flag[s] = keys[s] != CM_EMPTY ? 1 : 0;
}
// kept: live, or of an incarnation in the held list (n_held 0: live only)
__global__ void cm_live_kernel(const int* __restrict__ pt_slot, const int* __restrict__ pt_epoch, int n, const int* __restrict__ epoch, const unsigned long long* __restrict__ held,
                               int n_held, unsigned char* __restrict__ flag) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const int s = pt_slot[t];
  flag[t] = (s >= 0 && (pt_epoch[t] == epoch[s] || (n_held > 0 && cm_is_held(held, n_held, s, pt_epoch[t])))) ? 1 : 0;
}
// cur (NULL: none): the ordinal of every cell's current incarnation
__global__ void cm_export_cells_kernel(const unsigned long long* __restrict__ sorted_keys, const int* __restrict__ sorted_slots, int n, const int* __restrict__ create_frame,
                                       const int* __restrict__ last_update, ll_image_cell* __restrict__ out, const int* __restrict__ epoch,
                                       const unsigned long long* __restrict__ held, int n_held, int* __restrict__ cur) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const int s = sorted_slots[r];
  ll_image_cell c; c.key = sorted_keys[r]; c.create_frame = create_frame[s]; c.last_update = last_update[s];
  out[r] = c;
  if (cur) cur[r] = cm_ordinal(held, n_held, s, epoch[s]);
}
// ord (NULL: none): the ordinal of every point's incarnation
__global__ void cm_export_points_kernel(const float4* __restrict__ pts, const int* __restrict__ pt_slot, const int* __restrict__ idx, int n, const int* __restrict__ rank_of_slot,
                                        ll_image_cell_point* __restrict__ out, const int* __restrict__ pt_epoch, const unsigned long long* __restrict__ held, int n_held,
                                        int* __restrict__ ord) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const int t = idx[r]; const float4 p = pts[t];
  ll_image_cell_point o; o.x = p.x; o.y = p.y; o.z = p.z; o.cell = rank_of_slot[pt_slot[t]];
  out[r] = o;
  if (ord) ord[r] = cm_ordinal(held, n_held, pt_slot[t], pt_epoch[t]);
}
// one thread per cell: the probe sequence of cm_locate_kernel into an empty table (keys are distinct, so every CAS claims a fresh slot); cur (NULL:
// every epoch 0) the cells' epochs
__global__ void cm_import_cells_kernel(const ll_image_cell* __restrict__ in, int n, unsigned long long* keys, unsigned mask, int* create_frame, int* last_update, int* epoch, int* bump,
                                       int* __restrict__ slot_of_rank, const int* __restrict__ cur) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const ll_image_cell c = in[r];
  unsigned h = cm_hash(c.key, mask);
  while (atomicCAS(&keys[h], CM_EMPTY, c.key) != CM_EMPTY) h = (h + 1) & mask;
  create_frame[h] = c.create_frame; last_update[h] = c.last_update; epoch[h] = cur ? cur[r] : 0; bump[h] = -1;
  slot_of_rank[r] = (int)h;
}
// ord (NULL: every epoch 0) the points' epochs
__global__ void cm_import_points_kernel(const ll_image_cell_point* __restrict__ in, int n, const int* __restrict__ slot_of_rank, float4* __restrict__ pts, int* __restrict__ pt_slot,
                                        int* __restrict__ pt_epoch, const int* __restrict__ ord) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const ll_image_cell_point p = in[t];
  pts[t] = make_float4(p.x, p.y, p.z, 0.f); pt_slot[t] = slot_of_rank[p.cell]; pt_epoch[t] = ord ? ord[t] : 0;
}

// The export's scratch over a table of T slots and a store of N points; rec = the cells then the kept points, as the image holds them (with a
// held list: then the cells' current ordinals and the points' ordinals)
struct CmExport {
  size_t cub_bytes = 0;
  unsigned char* flag; int* slots; unsigned long long* keys; unsigned long long* keys2; int* slots2; int* rank; int* idx; int* cnt; char* cub_tmp; int4* rec;
  CmExport(int T, int N) {
    size_t cub_a = 0, cub_b = 0;
    cub::DeviceSelect::Flagged(nullptr, cub_a, cub::CountingInputIterator<int>(0), (unsigned char*)nullptr, (int*)nullptr, (int*)nullptr, T > N ? T : N);
    cub::DeviceRadixSort::SortPairs(nullptr, cub_b, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int*)nullptr, (int*)nullptr, T, 0, 64);
    cub_bytes = cub_a > cub_b ? cub_a : cub_b;
  }
  void layout(Carve& c, size_t T, size_t N, size_t n_rec) {
    flag = c.take<unsigned char>(T > N ? T : N); slots = c.take<int>(T); keys = c.take<unsigned long long>(T); keys2 = c.take<unsigned long long>(T);
    slots2 = c.take<int>(T); rank = c.take<int>(T); idx = c.take<int>(N); cnt = c.take<int>(16); cub_tmp = c.take<char>(cub_bytes); rec = c.take<int4>(n_rec);
  }
};
static size_t cm_export_rec(size_t n_cells, size_t n_pts, const CmHeld* held) { return n_cells + n_pts + (held ? (n_cells + n_pts + 3) / 4 : 0); }   // int4 records

// Cells in the table and live points in the store, the frame index and the out-of-range count (the map is only read)
int cm_count(ll_ctx* ctx, ll_cellmap* m, int* n_cells, int* n_live, int* frame_idx, int* n_out_of_range) {
  *frame_idx = m->current_frame_idx; *n_out_of_range = m->n_out_of_range;
  cudaStream_t s = ctx->stream;
  int* d = nullptr;
  LL_CUDA(ctx, ctx->scratch.carve([&](Carve& c) { d = c.take<int>(1); }));
  LL_CUDA(ctx, cudaMemsetAsync(d, 0, 4, s));
  if (m->n_pts > 0) { cm_count_alive_kernel<<<ll_div_up(m->n_pts, 256), 256, 0, s>>>(m->pt_slot, m->pt_epoch, m->n_pts, m->epoch, d); ctx->launches++; }
  int h[2] = {0, 0};
  LL_CUDA(ctx, cudaMemcpyAsync(h, m->d_counters, 4, cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaMemcpyAsync(h + 1, d, 4, cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  *n_cells = h[0]; *n_live = h[1];
  return LL_OK;
}

// The store indices of the kept points (live, and those of the held incarnations) in store order into a.idx (their count into a.cnt[1]), on the
// context's stream.
static int cm_select_live(ll_ctx* ctx, ll_cellmap* m, CmExport& a, const CmHeld* held = nullptr) {
  size_t cub_c = a.cub_bytes;
  const int N = m->n_pts;
  cm_live_kernel<<<ll_div_up(N, 256), 256, 0, ctx->stream>>>(m->pt_slot, m->pt_epoch, N, m->epoch, held ? held->ids : nullptr, held ? held->n : 0, a.flag);
  LL_CUDA(ctx, cub::DeviceSelect::Flagged(a.cub_tmp, cub_c, cub::CountingInputIterator<int>(0), a.flag, a.idx, a.cnt + 1, N, ctx->stream));
  ctx->launches += 2;
  return LL_OK;
}

// The kept points of a map with a held list (the count cm_export takes); the map is only read.
int cm_count_kept(ll_ctx* ctx, ll_cellmap* m, const CmHeld& held, int* n_kept) {
  *n_kept = 0;
  const int T = m->table_cap, N = m->n_pts;
  if (N == 0) return LL_OK;
  CmExport a(T, N);
  LL_CUDA(ctx, ctx->scratch.carve([&](Carve& c) { a.layout(c, T, N, 0); }));
  LL_TRY(cm_select_live(ctx, m, a, &held));
  LL_CUDA(ctx, cudaMemcpyAsync(n_kept, a.cnt + 1, 4, cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return LL_OK;
}

// The map's cells (ascending key) and live points (store order) into out: n_cells ll_image_cell then n_live ll_image_cell_point, the counts
// cm_count gave; with a held list also the points of the held incarnations, then int32 current ordinal[n_cells] and ordinal[n_live] (n_live:
// cm_count_kept's count).  One copy to the host; the map's buffers are only read.
int cm_export(ll_ctx* ctx, ll_cellmap* m, int n_cells, int n_live, void* out, const CmHeld* held) {
  cudaStream_t s = ctx->stream;
  const int T = m->table_cap, N = m->n_pts;
  if (n_cells + n_live == 0) return LL_OK;
  CmExport a(T, N);
  LL_CUDA(ctx, ctx->scratch.carve([&](Carve& c) { a.layout(c, T, N, cm_export_rec((size_t)n_cells, (size_t)n_live, held)); }));
  ll_image_cell* cells = (ll_image_cell*)a.rec; ll_image_cell_point* pts = (ll_image_cell_point*)(a.rec + n_cells);
  int* cur = held ? (int*)(a.rec + n_cells + n_live) : nullptr; int* ord = held ? cur + n_cells : nullptr;
  const unsigned long long* h_ids = held ? held->ids : nullptr; const int n_held = held ? held->n : 0;
  size_t cub_c = a.cub_bytes;
  LL_CUDA(ctx, cudaMemsetAsync(a.cnt, 0, 8, s));
  // cells: occupied slots, sorted by key, and the rank of every slot
  cm_occupied_kernel<<<ll_div_up(T, 256), 256, 0, s>>>(m->keys, T, a.flag);
  LL_CUDA(ctx, cub::DeviceSelect::Flagged(a.cub_tmp, cub_c, cub::CountingInputIterator<int>(0), a.flag, a.slots, a.cnt + 0, T, s));
  ctx->launches += 2;
  if (n_cells > 0) {
    cm_gather_keys_kernel<<<ll_div_up(n_cells, 256), 256, 0, s>>>(m->keys, a.slots, a.cnt + 0, a.keys);
    LL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(a.cub_tmp, cub_c, a.keys, a.keys2, a.slots, a.slots2, n_cells, 0, 64, s));
    cm_rank_kernel<<<ll_div_up(n_cells, 256), 256, 0, s>>>(a.slots2, n_cells, a.rank);
    cm_export_cells_kernel<<<ll_div_up(n_cells, 256), 256, 0, s>>>(a.keys2, a.slots2, n_cells, m->create_frame, m->last_update, cells, m->epoch, h_ids, n_held, cur);
    ctx->launches += 4;
  }
  // kept points in store order
  if (N > 0) {
    LL_TRY(cm_select_live(ctx, m, a, held));
    if (n_live > 0) {
      cm_export_points_kernel<<<ll_div_up(n_live, 256), 256, 0, s>>>(m->pts, m->pt_slot, a.idx, n_live, a.rank, pts, m->pt_epoch, h_ids, n_held, ord);
      ctx->launches++;
    }
  }
  LL_CUDA(ctx, cudaGetLastError());
  int h[2] = {0, 0};
  LL_CUDA(ctx, cudaMemcpyAsync(h, a.cnt, 8, cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaMemcpyAsync(out, a.rec, ((size_t)n_cells + n_live) * (held ? 20 : 16), cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  if (h[0] != n_cells || h[1] != n_live) { ctx->set_error("cell map changed while it was saved"); return LL_ERR_INVALID; }
  return LL_OK;
}

int cm_live_points(ll_ctx* ctx, ll_cellmap* m, int n_live, float4* dst) {
  const int T = m->table_cap, N = m->n_pts;
  if (n_live <= 0 || N <= 0) return LL_OK;
  CmExport a(T, N);
  LL_CUDA(ctx, ctx->scratch.carve([&](Carve& c) { a.layout(c, T, N, 0); }));
  LL_TRY(cm_select_live(ctx, m, a));
  LL_TRY(launch_gather_points(ctx, ctx->stream, m->pts, a.idx, n_live, dst));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // (a lives in the scratch arena, which the next carve may reallocate)
  return LL_OK;
}

// An empty map (just created) in the state of an exported one: in = n_cells ll_image_cell (ascending key) then n_live ll_image_cell_point,
// with incarnations then int32 current ordinal[n_cells] and ordinal[n_live] (set as the epochs), host memory, validated by the caller
// (distinct keys, ranks < n_cells, ordinals <= their cell's current one).  slot_of_rank (NULL: not wanted): each cell's slot, to the host.
int cm_import(ll_ctx* ctx, ll_cellmap* m, int frame_idx, int n_out_of_range, const void* in, int n_cells, int n_live, bool incarnations, int* slot_of_rank_out) {
  cudaStream_t s = ctx->stream;
  if (m->n_pts != 0 || m->n_cells != 0) { ctx->set_error("import into a cell map that is not empty"); return LL_ERR_INVALID; }
  if (n_cells > m->table_cap / 2) { ctx->set_error("cell table more than half full: create the map with a larger max_cells"); return LL_ERR_CAPACITY; }
  if (n_live > 0) LL_TRY(cm_reserve_store(ctx, m, n_live));
  int4* rec = nullptr; int* slot_of_rank = nullptr;
  const CmHeld none{nullptr, 0};
  const size_t n_rec = cm_export_rec((size_t)n_cells, (size_t)n_live, incarnations ? &none : nullptr);
  LL_CUDA(ctx, ctx->scratch.carve([&](Carve& c) { rec = c.take<int4>(n_rec); slot_of_rank = c.take<int>(n_cells); }));
  if (n_cells + n_live > 0) LL_CUDA(ctx, cudaMemcpyAsync(rec, in, ((size_t)n_cells + n_live) * (incarnations ? 20 : 16), cudaMemcpyHostToDevice, s));
  const int* cur = incarnations ? (const int*)(rec + n_cells + n_live) : nullptr; const int* ord = incarnations ? cur + n_cells : nullptr;
  if (n_cells > 0) {
    cm_import_cells_kernel<<<ll_div_up(n_cells, 256), 256, 0, s>>>((const ll_image_cell*)rec, n_cells, m->keys, (unsigned)(m->table_cap - 1), m->create_frame, m->last_update,
                                                                   m->epoch, m->bump, slot_of_rank, cur);
    ctx->launches++;
  }
  if (n_live > 0) {
    cm_import_points_kernel<<<ll_div_up(n_live, 256), 256, 0, s>>>((const ll_image_cell_point*)(rec + n_cells), n_live, slot_of_rank, m->pts, m->pt_slot, m->pt_epoch, ord);
    ctx->launches++;
  }
  if (slot_of_rank_out && n_cells > 0) LL_CUDA(ctx, cudaMemcpyAsync(slot_of_rank_out, slot_of_rank, (size_t)n_cells * 4, cudaMemcpyDeviceToHost, s));
  const int c[3] = {n_cells, 0, n_out_of_range};   // d_counters: cells, scratch, points out of the key's range so far
  LL_CUDA(ctx, cudaMemcpyAsync(m->d_counters, c, sizeof(c), cudaMemcpyHostToDevice, s));
  LL_CUDA(ctx, cudaGetLastError());
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  m->n_pts = n_live; m->n_cells = n_cells; m->current_frame_idx = frame_idx; m->n_out_of_range = n_out_of_range; m->generation++;
  return LL_OK;
}
