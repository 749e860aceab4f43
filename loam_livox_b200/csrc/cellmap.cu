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

#define CM_EMPTY 0xffffffffffffffffull
#define CM_BIAS (1 << 20)

struct ll_cellmap {
  int device = 0;
  float resolution = 0.5f;          // what set_resolution(r) stores: r / 2
  int revisit_threshold = 2147483647;
  int current_frame_idx = 0;
  int n_pts = 0, cap_pts = 0;       // used / allocated entries of the point store (dead points included until the next rebuild)
  int table_cap = 0;                // power of two
  unsigned long long* keys = nullptr; int* last_update = nullptr; int* create_frame = nullptr; int* epoch = nullptr; int* bump = nullptr;
  int* d_counters = nullptr;        // [0] number of cells, [1] scratch
  float4* pts = nullptr; int* pt_slot = nullptr; int* pt_epoch = nullptr;
  DevBuf table_buf, store_buf, store_alt, out_buf, tmp_buf;
};

__device__ __forceinline__ unsigned long long cm_pack(int k, int j, int i) {
  return ((unsigned long long)(unsigned)(k + CM_BIAS) << 42) | ((unsigned long long)(unsigned)(j + CM_BIAS) << 21) | (unsigned long long)(unsigned)(i + CM_BIAS);
}
__device__ __forceinline__ void cm_unpack(unsigned long long key, int& k, int& j, int& i) {
  k = (int)((key >> 42) & 0x1fffffull) - CM_BIAS; j = (int)((key >> 21) & 0x1fffffull) - CM_BIAS; i = (int)(key & 0x1fffffull) - CM_BIAS;
}
__device__ __forceinline__ unsigned cm_hash(unsigned long long key, unsigned mask) { return (unsigned)((key * 0x9E3779B97F4A7C15ull) >> 32) & mask; }

// pass 1: cell lookup / creation for every new point (find_cell with if_add = 1)
__global__ void cm_locate_kernel(const float4* __restrict__ in, int n, float box, float half, int cur, unsigned long long* keys, unsigned mask, int* create_frame, int* last_update,
                                 int* epoch, int* bump, int* counters, int* __restrict__ slot_out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const float4 p = in[t];
  if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) { slot_out[t] = -1; return; }
  const int i = (int)roundf((p.x - half) / box), j = (int)roundf((p.y - half) / box), k = (int)roundf((p.z - half) / box);
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
  const int bx = (int)floorf(ox * inv) - 2, by = (int)floorf(oy * inv) - 2, bz = (int)floorf(oz * inv) - 2;
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
  if (!ctx || !out || !(resolution > 0.f)) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  ll_cellmap* m = new ll_cellmap(); m->device = ctx->device; m->resolution = resolution * 0.5f; m->revisit_threshold = revisit_threshold;
  int cap = 1 << 12; while (cap < 2 * (max_cells > 0 ? max_cells : (1 << 20))) cap <<= 1;
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
  const bool first = m->current_frame_idx == 0 && m->n_pts == 0;
  if (n > 0) {
    LL_TRY(cm_reserve_store(ctx, m, m->n_pts + (int)n));
    CmAppend ap; LL_CUDA(ctx, m->tmp_buf.carve([&](Carve& c) { ap.layout(c, n); }));
    float4* d_in = ap.in; int* d_slot = ap.slot;
    LL_TRY(upload_cloud(ctx, pts, n, fmt, where, d_in));
    const float box = m->resolution * 1.0f, half = m->resolution * 0.5f;
    const int blocks = ll_div_up((int)n, 256), cur = m->current_frame_idx;
    cm_locate_kernel<<<blocks, 256, 0, s>>>(d_in, (int)n, box, half, cur, m->keys, (unsigned)(m->table_cap - 1), m->create_frame, m->last_update, m->epoch, m->bump, m->d_counters, d_slot);
    cm_revisit_kernel<<<blocks, 256, 0, s>>>(d_slot, (int)n, cur, m->revisit_threshold, m->create_frame, m->last_update, m->epoch, m->bump);
    cm_store_kernel<<<blocks, 256, 0, s>>>(d_in, d_slot, (int)n, cur, m->n_pts, m->epoch, m->bump, m->create_frame, m->last_update, m->pts, m->pt_slot, m->pt_epoch);
    ctx->launches += 3;
    LL_CUDA(ctx, cudaGetLastError());
    m->n_pts += (int)n;
    int cells = 0;
    LL_CUDA(ctx, cudaMemcpyAsync(&cells, m->d_counters, 4, cudaMemcpyDeviceToHost, s));
    LL_CUDA(ctx, cudaStreamSynchronize(s));
    if (cells > m->table_cap / 2) { ctx->set_error("cell table more than half full: create the map with a larger max_cells"); return LL_ERR_CAPACITY; }
  }
  if (first) m->current_frame_idx++;   // set_point_cloud() bumps the frame index too (:616) ...
  m->current_frame_idx++;              // ... and append_cloud() always does (:666)
  return LL_OK;
}

// update_buff_for_matching, matching_mode 1, for one map (laser_mapping.hpp:475-516).  The assembled cloud stays on the device
// (*out_dev, valid until the next call on this map); it is also copied to out_host when that is not NULL (cap points).
int ll_cellmap_assemble(ll_ctx* ctx, ll_cellmap* m, const double q_wxyz[4], const double t[3], float search_range, float fov_deg, float leaf, int down_sample_replace,
                        ll_point* out_host, size_t cap, size_t* n_out, int* cells_in_fov, const ll_point** out_dev) {
  if (!ctx || !m || !q_wxyz || !t || !n_out || !(leaf > 0.f)) return LL_ERR_INVALID;
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
    m->pts = np; m->pt_slot = ns; m->pt_epoch = ne; m->cap_pts = cap_new; m->n_pts = n_new;
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
