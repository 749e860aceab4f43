// Cloud plumbing kernels: format repack, pointAssociateToMap over a cloud, VoxelGrid down-sampling.
//
// Replaces, on the reference side:
//   pcl::VoxelGrid<PointXYZI>::filter (third-party PCL, restated)  call sites loam_livox/source/laser_feature_extractor.hpp:372-380,
//                                   loam_livox/source/laser_mapping.hpp:491,509,533-537,1367-1373,1434-1437                 (K4)
//   pointcloudAssociateToMap        loam_livox/source/point_cloud_registration.hpp:622-661,673-685                           (K6, cloud form)
//
// Compiled with -fmad=false (voxel indices, centroids and the transform must round like the scalar CPU code).
#include <algorithm>
#include <cooperative_groups.h>
#include <cub/cub.cuh>
#include "common.cuh"
#include "kernels.cuh"
#include "exact_math.cuh"

#define FULL 0xffffffffu
namespace cg = cooperative_groups;

// ------------------------------------------------------------------------------------------------ upload / repack
__global__ void repack_pcl32_kernel(const float* __restrict__ src, int n, float4* __restrict__ dst) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 a = reinterpret_cast<const float4*>(src)[2 * i];      // x y z pad
  const float4 b = reinterpret_cast<const float4*>(src)[2 * i + 1];  // intensity pad pad pad
  dst[i] = make_float4(a.x, a.y, a.z, b.x);
}

// LL_FMT_STRIDED: byte-wise little-endian loads (the offsets of a PointCloud2 record need not be aligned)
__device__ __forceinline__ float load_f32_le(const unsigned char* p) { const unsigned v = (unsigned)p[0] | ((unsigned)p[1] << 8) | ((unsigned)p[2] << 16) | ((unsigned)p[3] << 24); return __uint_as_float(v); }
__global__ void repack_strided_kernel(const unsigned char* __restrict__ src, int n, ll_point_layout L, float4* __restrict__ dst) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned char* r = src + (size_t)i * L.point_step;
  float it = 0.f;
  if (L.intensity_datatype == LL_I_FLOAT32) it = load_f32_le(r + L.offset_intensity);
  else if (L.intensity_datatype == LL_I_UINT8) it = (float)r[L.offset_intensity];
  else if (L.intensity_datatype == LL_I_UINT16) it = (float)((unsigned)r[L.offset_intensity] | ((unsigned)r[L.offset_intensity + 1] << 8));
  dst[i] = make_float4(load_f32_le(r + L.offset_x), load_f32_le(r + L.offset_y), load_f32_le(r + L.offset_z), it);
}

// The other direction (pcl::toROSMsg, laser_feature_extractor.hpp:367-384): 16-byte points -> records of a sensor_msgs/PointCloud2 payload.
// Bytes of a record that belong to no field are zeroed.
__device__ __forceinline__ void store_f32_le(unsigned char* p, float f) { const unsigned v = __float_as_uint(f); p[0] = v & 255; p[1] = (v >> 8) & 255; p[2] = (v >> 16) & 255; p[3] = v >> 24; }
__global__ void pack_strided_kernel(const float4* __restrict__ src, int n, ll_point_layout L, unsigned char* __restrict__ dst) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned char* r = dst + (size_t)i * L.point_step;
  for (int b = 0; b < L.point_step; b++) r[b] = 0;
  const float4 p = src[i];
  store_f32_le(r + L.offset_x, p.x); store_f32_le(r + L.offset_y, p.y); store_f32_le(r + L.offset_z, p.z);
  if (L.intensity_datatype == LL_I_FLOAT32) store_f32_le(r + L.offset_intensity, p.w);
  else if (L.intensity_datatype == LL_I_UINT8) r[L.offset_intensity] = (unsigned char)fminf(fmaxf(p.w, 0.f), 255.f);
  else if (L.intensity_datatype == LL_I_UINT16) { const unsigned v = (unsigned)fminf(fmaxf(p.w, 0.f), 65535.f); r[L.offset_intensity] = v & 255; r[L.offset_intensity + 1] = v >> 8; }
}
int launch_pack_strided(ll_ctx* ctx, const float4* d_src, int n, unsigned char* d_dst) {
  if (n == 0) return LL_OK;
  pack_strided_kernel<<<ll_div_up(n, 256), 256, 0, ctx->stream>>>(d_src, n, ctx->layout, d_dst); ctx->launches++;
  LL_CUDA(ctx, cudaGetLastError());
  return LL_OK;
}

int upload_cloud(ll_ctx* ctx, cudaStream_t s, const void* src, size_t n, int fmt, int where, float4* d_dst) {
  if (n == 0) return LL_OK;
  if (fmt == LL_FMT_XYZI16) {
    LL_CUDA(ctx, cudaMemcpyAsync(d_dst, src, n * 16, where == LL_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s));
  } else if (fmt == LL_FMT_PCL32) {
    const float* d_src = (const float*)src;
    if (where == LL_HOST) {
      LL_CUDA(ctx, ctx->stage_in.reserve(n * 32));
      LL_CUDA(ctx, cudaMemcpyAsync(ctx->stage_in.p, src, n * 32, cudaMemcpyHostToDevice, s));
      d_src = ctx->stage_in.as<float>();
    }
    repack_pcl32_kernel<<<ll_div_up((int)n, 256), 256, 0, s>>>(d_src, (int)n, d_dst); ctx->launches++;
    LL_CUDA(ctx, cudaGetLastError());
  } else if (fmt == LL_FMT_STRIDED) {
    const ll_point_layout L = ctx->layout;
    const unsigned char* d_src = (const unsigned char*)src;
    if (where == LL_HOST) {
      LL_CUDA(ctx, ctx->stage_in.reserve(n * (size_t)L.point_step));
      LL_CUDA(ctx, cudaMemcpyAsync(ctx->stage_in.p, src, n * (size_t)L.point_step, cudaMemcpyHostToDevice, s));
      d_src = ctx->stage_in.as<unsigned char>();
    }
    repack_strided_kernel<<<ll_div_up((int)n, 256), 256, 0, s>>>(d_src, (int)n, L, d_dst); ctx->launches++;
    LL_CUDA(ctx, cudaGetLastError());
  } else { ctx->set_error("unknown point format"); return LL_ERR_INVALID; }
  return LL_OK;
}

// ------------------------------------------------------------------------------------------------ transform
__global__ void transform_kernel(const double* __restrict__ pose7, const float4* __restrict__ in, int n, const int* __restrict__ d_n, float4* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (d_n) n = min(n, *d_n);
  if (i >= n) return;
  const float4 p = in[i];
  double q[4] = {pose7[0], pose7[1], pose7[2], pose7[3]};
  double wx, wy, wz; qrot_d(q, (double)p.x, (double)p.y, (double)p.z, wx, wy, wz);
  out[i] = make_float4((float)(wx + pose7[4]), (float)(wy + pose7[5]), (float)(wz + pose7[6]), p.w);
}
int launch_transform(ll_ctx* ctx, cudaStream_t s, const double* d_pose7, const float4* d_in, int n, float4* d_out) {
  if (n == 0) return LL_OK;
  transform_kernel<<<ll_div_up(n, 256), 256, 0, s>>>(d_pose7, d_in, n, nullptr, d_out); ctx->launches++;
  LL_CUDA(ctx, cudaGetLastError());
  return LL_OK;
}

// ------------------------------------------------------------------------------------------------ VoxelGrid
// One pass filters nseg disjoint contiguous segments of the input, each exactly as a VoxelGrid of that segment alone: segment s is
// [end[s - 1], end[s]) (end[-1] = 0; every end clamped to n_cap; end == null: one segment of n_cap points).  Each segment gets its own bounds,
// grid and int32-overflow decision; the segment id sits above the 32 voxel-key bits of the sort key, so equal voxels of two segments never
// merge and, the radix sort being stable, every voxel still sums its points in ascending input order.  The outputs follow one another:
// segment s's voxels are out[out_end[s - 1], out_end[s]).  One segment sorts 32-bit keys, as a single-cloud VoxelGrid always did.
struct VgMeta {
  int mn[3], mx[3];     // ordered-int encodings of the float min / max
  int n_finite;
  int passthrough;      // dx*dy*dz overflows int32: PCL warns and copies the input through
  int n_in, begin;      // the segment's input range
  int min_b[3]; int mul[3];
  float inv;
  int ticket;           // blocks of the segment's row of vg_minmax_setup_kernel that have finished (the last one does the set-up and resets it)
};
struct VgSegs {
  const int* end; int nseg, n_cap;
  __device__ __forceinline__ int end_of(int s) const { return end ? min(end[s], n_cap) : n_cap; }
  __device__ __forceinline__ int begin_of(int s) const { return s ? min(end_of(s - 1), end_of(s)) : 0; }
  __device__ __forceinline__ int find(int i) const {   // segment holding input index i (nseg: past the last segment)
    if (nseg == 1) return i < end_of(0) ? 0 : 1;
    int lo = 0, hi = nseg;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (i < end_of(mid)) hi = mid; else lo = mid + 1; }
    return lo;
  }
};
template <typename K> __device__ __forceinline__ unsigned vg_low(K k) { return (unsigned)(k & 0xffffffffu); }
template <typename K> __device__ __forceinline__ int vg_seg(K k) { return sizeof(K) == 4 ? 0 : (int)((unsigned long long)k >> 32); }

// Min / max over the finite points of segment blockIdx.y, then -- by the last block of that segment to finish -- the grid set-up of
// VoxelGrid::applyFilter (one launch instead of init + minmax + setup; `m` is cleared by a memset node: mins are kept as the bitwise complement
// of their order-preserving key, so that "all zero" is the neutral element of the atomicMax that reduces both the mins and the maxs).
__device__ __forceinline__ unsigned f2key(float f) { return (unsigned)ll_f2ord(f) ^ 0x80000000u; }     // unsigned order == float order
__device__ __forceinline__ float key2f(unsigned k) { return ll_ord2f((int)(k ^ 0x80000000u)); }
// The grid set-up of VoxelGrid::applyFilter from the bounds mn / mx of the finite points (any: there is at least one).
__device__ __forceinline__ void vg_grid(VgMeta* m, bool any, const float* mn, const float* mx, float leaf) {
  m->passthrough = 0;
  const float inv = 1.0f / leaf; m->inv = inv;
  if (!any) { for (int k = 0; k < 3; k++) { m->min_b[k] = 0; m->mul[k] = 0; } return; }
  long long dx = (long long)((mx[0] - mn[0]) * inv) + 1, dy = (long long)((mx[1] - mn[1]) * inv) + 1, dz = (long long)((mx[2] - mn[2]) * inv) + 1;
  if (dx * dy * dz > 2147483647LL) { m->passthrough = 1; return; }
  int div_b[3];
  for (int k = 0; k < 3; k++) { m->min_b[k] = (int)floorf(mn[k] * inv); int max_b = (int)floorf(mx[k] * inv); div_b[k] = max_b - m->min_b[k] + 1; }
  m->mul[0] = 1; m->mul[1] = div_b[0]; m->mul[2] = div_b[0] * div_b[1];
}
// Voxel key of a point (wrapping int arithmetic, as the scalar code); 0xffffffff for a non-finite point.
__device__ __forceinline__ unsigned vg_key(const float4 p, const VgMeta& m) {
  if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) return 0xffffffffu;
  const float inv = m.inv;
  int ijk0 = (int)(floorf(p.x * inv) - (float)m.min_b[0]);
  int ijk1 = (int)(floorf(p.y * inv) - (float)m.min_b[1]);
  int ijk2 = (int)(floorf(p.z * inv) - (float)m.min_b[2]);
  return (unsigned)(ijk0 * m.mul[0] + ijk1 * m.mul[1] + ijk2 * m.mul[2]);
}
__global__ void vg_minmax_setup_kernel(const float4* __restrict__ in, VgMeta* metas, VgSegs g, float leaf) {
  VgMeta* m = metas + blockIdx.y;
  const int b = g.begin_of(blockIdx.y), n = g.end_of(blockIdx.y);
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY}; int cnt = 0;
  for (int i = b + blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float4 p = in[i];
    if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
      lo[0] = fminf(lo[0], p.x); lo[1] = fminf(lo[1], p.y); lo[2] = fminf(lo[2], p.z);
      hi[0] = fmaxf(hi[0], p.x); hi[1] = fmaxf(hi[1], p.y); hi[2] = fmaxf(hi[2], p.z); cnt++;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int k = 0; k < 3; k++) { lo[k] = fminf(lo[k], __shfl_xor_sync(FULL, lo[k], o)); hi[k] = fmaxf(hi[k], __shfl_xor_sync(FULL, hi[k], o)); }
    cnt += __shfl_xor_sync(FULL, cnt, o);
  }
  if ((threadIdx.x & 31) == 0 && cnt > 0) {
#pragma unroll
    for (int k = 0; k < 3; k++) { atomicMax((unsigned*)&m->mn[k], ~f2key(lo[k])); atomicMax((unsigned*)&m->mx[k], f2key(hi[k])); }
    atomicAdd(&m->n_finite, cnt);
  }
  __threadfence();
  __syncthreads();
  __shared__ int s_last;
  if (threadIdx.x == 0) s_last = (atomicAdd(&m->ticket, 1) == (int)gridDim.x - 1) ? 1 : 0;
  __syncthreads();
  if (!s_last || threadIdx.x != 0) return;
  __threadfence();
  // ---- set-up (the last block sees every block's contribution)
  volatile VgMeta* v = m;
  m->n_in = n - b; m->begin = b; m->ticket = 0;
  float mn[3], mx[3]; for (int k = 0; k < 3; k++) { mn[k] = key2f(~(unsigned)v->mn[k]); mx[k] = key2f((unsigned)v->mx[k]); }
  vg_grid(m, v->n_finite > 0, mn, mx, leaf);
}
// Sort key of input index i: the segment id above the 32 voxel-key bits (K = 32-bit: one segment).  Non-finite points take the low word
// 0xffffffff (the end of their segment), points past the last segment the largest key.  A pass-through segment keys every point by its
// position, so that each one is a voxel of its own and the centroid kernel copies it.
template <typename K>
__global__ void vg_keys_kernel(const float4* __restrict__ in, const VgMeta* __restrict__ metas, VgSegs g, K* __restrict__ keys, int* __restrict__ vals) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.n_cap) return;
  const int s = g.find(i);
  unsigned key = 0xffffffffu;
  if (s < g.nseg) {
    const VgMeta* m = metas + s;
    key = m->passthrough ? (unsigned)(i - m->begin) : vg_key(in[i], *m);
  }
  keys[i] = sizeof(K) == 4 ? (K)key : (K)(((unsigned long long)s << 32) | key);
  vals[i] = i;
}
// First element of every run of equal (valid) keys in the sorted key array: the predicate of the stream compaction that lists the voxels.
template <typename K> struct VgHead {
  const K* keys;
  __device__ __forceinline__ bool operator()(int i) const { const K k = keys[i]; return vg_low(k) != 0xffffffffu && (i == 0 || keys[i - 1] != k); }
};
// One thread per voxel: sequential float sum in ascending input index (radix sort is stable), like CentroidPoint<PointXYZI>.  Voxel v of the
// whole pass is output v; out_end[s] = the voxels of segments 0..s (one thread per segment of block 0 finds it by bisection).
template <typename K>
__global__ void vg_centroid_kernel(const float4* __restrict__ in, const VgMeta* __restrict__ metas, int nseg, const K* __restrict__ keys, const int* __restrict__ vals,
                                   const int* __restrict__ heads, const int* __restrict__ d_num_heads, float4* __restrict__ out, int* __restrict__ out_end) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  const int nh = *d_num_heads;
  if (blockIdx.x == 0 && threadIdx.x < nseg) {
    int e = nh;
    if (sizeof(K) == 8) {   // first voxel of a later segment
      int lo = 0, hi = nh;
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (vg_seg(keys[heads[mid]]) > (int)threadIdx.x) hi = mid; else lo = mid + 1; }
      e = lo;
    }
    out_end[threadIdx.x] = e;
  }
  if (v >= nh) return;
  const int b = heads[v];
  const VgMeta* m = metas + vg_seg(keys[b]);
  if (m->passthrough) { out[v] = in[vals[b]]; return; }
  const int e = min(v + 1 < nh ? heads[v + 1] : 0x7fffffff, m->begin + m->n_finite);
  float sx = 0.f, sy = 0.f, sz = 0.f, si = 0.f;
  for (int li = b; li < e; li++) { const float4 p = in[vals[li]]; sx += p.x; sy += p.y; sz += p.z; si += p.w; }
  const float cnt = (float)(e - b);
  out[v] = make_float4(sx / cnt, sy / cnt, sz / cnt, si / cnt);
}

static int vg_sort_bits(int nseg) { int b = 32; if (nseg > 1) for (int v = nseg; v > 0; v >>= 1) b++; return b; }   // segment ids 0..nseg
// The scratch of one VoxelGrid pass over n_cap points (n_cap > 0) in nseg segments.
template <typename K> struct VgScratch {
  size_t sort_bytes = 0, sel_bytes = 0;
  VgMeta* meta; int* d_num_heads; K* k0; K* k1; int* v0; int* v1; int* heads; char* tmp;
  VgScratch(int n_cap, int nseg) {
    cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (K*)nullptr, (K*)nullptr, (int*)nullptr, (int*)nullptr, n_cap, 0, vg_sort_bits(nseg));
    cub::DeviceSelect::If(nullptr, sel_bytes, cub::CountingInputIterator<int>(0), (int*)nullptr, (int*)nullptr, n_cap, VgHead<K>{nullptr});
  }
  void layout(Carve& c, int n_cap, int nseg) {
    meta = c.take<VgMeta>(nseg); d_num_heads = c.take<int>(1);
    k0 = c.take<K>(n_cap); k1 = c.take<K>(n_cap); v0 = c.take<int>(n_cap); v1 = c.take<int>(n_cap); heads = c.take<int>(n_cap);
    tmp = c.take<char>(sort_bytes > sel_bytes ? sort_bytes : sel_bytes);
  }
};
size_t voxel_grid_bytes(int n_cap, int nseg) {
  if (n_cap <= 0) return 0;
  if (nseg > 1) { VgScratch<unsigned long long> v(n_cap, nseg); return layout_bytes([&](Carve& c) { v.layout(c, n_cap, nseg); }); }
  VgScratch<unsigned> v(n_cap, 1);
  return layout_bytes([&](Carve& c) { v.layout(c, n_cap, 1); });
}
template <typename K>
static int voxel_grid_pass(ll_ctx* ctx, cudaStream_t s, DevBuf& scratch, const float4* d_in, int n_cap, const int* d_end, int nseg, float leaf, float4* d_out, int* d_out_end) {
  VgScratch<K> v(n_cap, nseg);
  LL_CUDA(ctx, scratch.carve([&](Carve& c) { v.layout(c, n_cap, nseg); }));
  const int blocks = ll_div_up(n_cap, 256);
  const VgSegs g{d_end, nseg, n_cap};
  LL_CUDA(ctx, cudaMemsetAsync(v.meta, 0, nseg * sizeof(VgMeta), s));
  vg_minmax_setup_kernel<<<dim3(min(blocks, ctx->num_sms * 2), nseg), 256, 0, s>>>(d_in, v.meta, g, leaf);
  vg_keys_kernel<K><<<blocks, 256, 0, s>>>(d_in, v.meta, g, v.k0, v.v0);
  LL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(v.tmp, v.sort_bytes, v.k0, v.k1, v.v0, v.v1, n_cap, 0, vg_sort_bits(nseg), s));
  LL_CUDA(ctx, cub::DeviceSelect::If(v.tmp, v.sel_bytes, cub::CountingInputIterator<int>(0), v.heads, v.d_num_heads, n_cap, VgHead<K>{v.k1}, s));
  vg_centroid_kernel<K><<<blocks, 256, 0, s>>>(d_in, v.meta, nseg, v.k1, v.v1, v.heads, v.d_num_heads, d_out, d_out_end);
  // minmax+setup, keys, radix sort (histogram, scan, one onesweep pass per 8 key bits), select (init, sweep), centroid
  ctx->launches += 7 + (uint64_t)(vg_sort_bits(nseg) + 7) / 8;
  LL_CUDA(ctx, cudaGetLastError());
  return LL_OK;
}
// On an explicit stream with its own scratch arena: VoxelGrid chains run side by side (every kernel here is far too small to fill the GPU,
// so the chains overlap almost perfectly).
int launch_voxel_grid_segments(ll_ctx* ctx, cudaStream_t s, DevBuf& scratch, const float4* d_in, int n_cap, const int* d_end, int nseg, float leaf, float4* d_out, int* d_out_end) {
  if (nseg < 1) return LL_OK;
  if (n_cap <= 0) { LL_CUDA(ctx, cudaMemsetAsync(d_out_end, 0, nseg * sizeof(int), s)); return LL_OK; }
  if (nseg == 1) return voxel_grid_pass<unsigned>(ctx, s, scratch, d_in, n_cap, d_end, 1, leaf, d_out, d_out_end);
  return voxel_grid_pass<unsigned long long>(ctx, s, scratch, d_in, n_cap, d_end, nseg, leaf, d_out, d_out_end);
}

// ------------------------------------------------------------------------------------------------ VoxelGrid chains in one cluster
// A chain of VoxelGrids (each on the previous one's output) run by one cluster of VGC_CTAS CTAs from the device count, without a host read:
// bounds (cluster reduction), set-up (vg_grid), keys (vg_key), a stable LSD radix sort of (key, input index) in distributed shared memory,
// the voxel heads and the centroids.  Position p of the sorted order lives in CTA p / per at p % per (per = ceil(count / VGC_CTAS)).
// The whole chain is latency-bound (a C2 scan's surface chain sorts under 100k keys): 16 SMs halve every CTA's share of the serial work
// against a portable cluster of 8, and the per-CTA footprint (about 147 KB of shared memory, 512 threads of 64 registers) still leaves room
// for a solver CTA on every SM the cluster occupies (the front end runs under the registration of the previous input).
#define VGC_CTAS 16
#define VGC_THREADS 512
#define VGC_WARPS (VGC_THREADS / 32)
#define VGC_PER_CTA 6400
#define VG_CLUSTER_CAP (VGC_CTAS * VGC_PER_CTA)   // largest host-known input count that takes the cluster path
#define VGC_RADIX 256                             // 8-bit digits: passes = ceil(bits of the largest key / 8)
struct VgcShared {
  unsigned idx[2][VGC_PER_CTA];         // input indices in position order (the sort's ping-pong buffers)
  unsigned key[2][VGC_PER_CTA];         // their keys (0xffffffff: dropped, before pass 0 only)
  unsigned kbuf[VGC_PER_CTA];           // per element: (digit << 16 | rank among the equal digits of its warp's segment)
  unsigned cnt[VGC_WARPS][VGC_RADIX];   // per warp and digit: count, then the warp's offset within the CTA
  unsigned hist[VGC_RADIX];             // the CTA's digit counts (read by the cluster)
  unsigned off[VGC_RADIX];              // the CTA's first position of each digit
  unsigned red[VGC_WARPS][8];
  unsigned bounds[7];                   // published: min keys, max keys (f2key) and count of the CTA's finite points
  unsigned keyinfo[2];                  // published: the CTA's kept points and the OR of their keys
  unsigned n_heads;                     // published
  int g_n, g_or, vbase, total;
  VgMeta meta;
  VgChainDev chain;                     // this cluster's chain (read where needed: no registers are left to hold its pointers over the sort)
  float4* out; int* d_n_out;            // the current VoxelGrid's
};
// Exclusive prefix sum of v over the CTA's threads in thread order; *total = the sum.
__device__ __forceinline__ unsigned vgc_scan(VgcShared& sh, unsigned v, unsigned* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const unsigned y = __shfl_up_sync(FULL, x, o); if (lane >= o) x += y; }
  if (lane == 31) sh.red[w][0] = x;
  __syncthreads();
  if (w == 0) {
    unsigned y = lane < VGC_WARPS ? sh.red[lane][0] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned z = __shfl_up_sync(FULL, y, o); if (lane >= o) y += z; }
    if (lane < VGC_WARPS) sh.red[lane][1] = y;
  }
  __syncthreads();
  const unsigned r = (w ? sh.red[w - 1][1] : 0) + x - v;
  *total = sh.red[VGC_WARPS - 1][1];
  __syncthreads();
  return r;
}
// VoxelGrid v of the cluster's chain on n points, by the whole cluster; *d_n_out[v] (CTA 0) and the return value: the output count.  Ends with a cluster
// barrier: the outputs are visible to the cluster and no CTA reads another's shared memory of this VoxelGrid afterwards.
extern __shared__ __align__(16) unsigned char vgc_smem[];
__device__ __forceinline__ int vgc_voxel_grid(int v, int n) {
  VgcShared& sh = *reinterpret_cast<VgcShared*>(vgc_smem);
  cg::cluster_group cl = cg::this_cluster();
  const float4* in = v ? sh.chain.out[0] : sh.chain.in;
  const int c = (int)cl.block_rank(), tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  if (tid == 0) { sh.out = sh.chain.out[v]; sh.d_n_out = sh.chain.d_n_out[v]; }   // published by the first __syncthreads below
  const int per_in = (n + VGC_CTAS - 1) / VGC_CTAS, i0 = min(n, c * per_in), l_in = min(n, i0 + per_in) - i0;   // this CTA's input slice
  // ---- bounds of the finite points: order-preserving keys reduce exactly in any order
  unsigned lo[3] = {~0u, ~0u, ~0u}, hi[3] = {0u, 0u, 0u}, nf = 0;
#pragma unroll 4
  for (int e = tid; e < l_in; e += VGC_THREADS) {
    const float4 p = __ldcg(in + i0 + e);
    if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
      const unsigned k[3] = {f2key(p.x), f2key(p.y), f2key(p.z)};
      for (int j = 0; j < 3; j++) { lo[j] = min(lo[j], k[j]); hi[j] = max(hi[j], k[j]); }
      nf++;
    }
  }
  for (int j = 0; j < 3; j++) { lo[j] = __reduce_min_sync(FULL, lo[j]); hi[j] = __reduce_max_sync(FULL, hi[j]); }
  nf = __reduce_add_sync(FULL, nf);
  if (lane == 0) { for (int j = 0; j < 3; j++) { sh.red[w][j] = lo[j]; sh.red[w][3 + j] = hi[j]; } sh.red[w][6] = nf; }
  __syncthreads();
  if (tid < 7) {
    unsigned r = sh.red[0][tid];
#pragma unroll 1
    for (int u = 1; u < VGC_WARPS; u++) { const unsigned x = sh.red[u][tid]; r = tid < 3 ? min(r, x) : tid < 6 ? max(r, x) : r + x; }
    sh.bounds[tid] = r;
  }
  cl.sync();
  if (w == 0) {   // every CTA sets up the same grid from the same bounds: lane r reads CTA r's
    unsigned b[7] = {~0u, ~0u, ~0u, 0u, 0u, 0u, 0u};
    if (lane < VGC_CTAS) { const unsigned* o = cl.map_shared_rank(sh.bounds, lane); for (int j = 0; j < 7; j++) b[j] = o[j]; }
    for (int j = 0; j < 3; j++) { b[j] = __reduce_min_sync(FULL, b[j]); b[3 + j] = __reduce_max_sync(FULL, b[3 + j]); }
    b[6] = __reduce_add_sync(FULL, b[6]);
    if (lane == 0) {
      float mn[3], mx[3]; for (int j = 0; j < 3; j++) { mn[j] = key2f(b[j]); mx[j] = key2f(b[3 + j]); }
      sh.meta.n_finite = (int)b[6];
      vg_grid(&sh.meta, b[6] > 0, mn, mx, sh.chain.leaf[v]);
    }
  }
  __syncthreads();
  if (sh.meta.passthrough) {   // PCL's int32 overflow: every point copied through, in input order
    float4* out = sh.out;
#pragma unroll 4
    for (int e = tid; e < l_in; e += VGC_THREADS) out[i0 + e] = __ldcg(in + i0 + e);
    if (c == 0 && tid == 0) *sh.d_n_out = n;
    cl.sync();
    return n;
  }
  // ---- keys of the slice (0xffffffff: dropped), the kept count and the OR of the kept keys
  unsigned any = 0, nk = 0;
#pragma unroll 2
  for (int e = tid; e < l_in; e += VGC_THREADS) {
    const unsigned k = vg_key(__ldcg(in + i0 + e), sh.meta);
    sh.key[1][e] = k;
    if (k != 0xffffffffu) { any |= k; nk++; }
  }
  any = __reduce_or_sync(FULL, any); nk = __reduce_add_sync(FULL, nk);
  if (lane == 0) { sh.red[w][0] = nk; sh.red[w][1] = any; }
  __syncthreads();
  if (tid == 0) {
    unsigned a = 0, s = 0; for (int u = 0; u < VGC_WARPS; u++) { s += sh.red[u][0]; a |= sh.red[u][1]; }
    sh.keyinfo[0] = s; sh.keyinfo[1] = a;
  }
  cl.sync();
  if (w == 0) {
    unsigned a = 0, s = 0;
    if (lane < VGC_CTAS) { const unsigned* o = cl.map_shared_rank(sh.keyinfo, lane); s = o[0]; a = o[1]; }
    s = __reduce_add_sync(FULL, s); a = __reduce_or_sync(FULL, a);
    if (lane == 0) { sh.g_n = (int)s; sh.g_or = (int)a; }
  }
  __syncthreads();
  const int nv = sh.g_n;
  if (nv == 0) {
    if (c == 0 && tid == 0) *sh.d_n_out = 0;
    cl.sync();
    return 0;
  }
  const int per = (nv + VGC_CTAS - 1) / VGC_CTAS, len = min(max(nv - c * per, 0), per);   // positions of this CTA after pass 0
  const int passes = max(1, (32 - __clz(sh.g_or) + 7) / 8);
  // ---- stable LSD radix sort: pass 0 reads the slice in input order (dropping the dropped points), every pass scatters (key, index) into the
  // owning CTA
#pragma unroll 1
  for (int pass = 0; pass < passes; pass++) {
    const int shift = 8 * pass;
    const unsigned* src = sh.idx[(pass + 1) & 1];
    const unsigned* ksrc = sh.key[(pass + 1) & 1];
    const int l = pass ? len : l_in, seg = (l + VGC_WARPS - 1) / VGC_WARPS, s0 = min(l, w * seg), s1 = min(l, s0 + seg);
    for (int d = lane; d < VGC_RADIX; d += 32) sh.cnt[w][d] = 0;
    __syncwarp();
    // rank of every element among the equal digits of its warp's segment, in order
#pragma unroll 1
    for (int b = s0; b < s1; b += 32) {
      const int e = b + lane;
      const unsigned k = e < s1 ? ksrc[e] : 0xffffffffu;
      const bool keep = k != 0xffffffffu;
      const unsigned d = (k >> shift) & (VGC_RADIX - 1);
      const unsigned peers = __match_any_sync(FULL, keep ? d : 0xffffffffu);
      const unsigned before = keep ? sh.cnt[w][d] : 0;
      __syncwarp();
      if (keep && lane == __ffs(peers) - 1) sh.cnt[w][d] = before + __popc(peers);
      if (e < s1) sh.kbuf[e] = keep ? (d << 16) | (before + __popc(peers & ((1u << lane) - 1))) : 0xffffffffu;
      __syncwarp();
    }
    __syncthreads();
    if (tid < VGC_RADIX) {
      unsigned run = 0;
      for (int u = 0; u < VGC_WARPS; u++) { const unsigned t = sh.cnt[u][tid]; sh.cnt[u][tid] = run; run += t; }
      sh.hist[tid] = run;
    }
    cl.sync();
    unsigned tot = 0, before = 0;
    if (tid < VGC_RADIX)
#pragma unroll 4
      for (int r = 0; r < VGC_CTAS; r++) { const unsigned h = cl.map_shared_rank(sh.hist, r)[tid]; tot += h; if (r < c) before += h; }
    unsigned all;
    const unsigned ex = vgc_scan(sh, tid < VGC_RADIX ? tot : 0u, &all);
    if (tid < VGC_RADIX) sh.off[tid] = ex + before;
    __syncthreads();
    unsigned* dst = sh.idx[pass & 1];
    unsigned* kdst = sh.key[pass & 1];
#pragma unroll 1
    for (int e = s0 + lane; e < s1; e += 32) {
      const unsigned pk = sh.kbuf[e];
      if (pk == 0xffffffffu) continue;
      const unsigned d = pk >> 16;
      const int pos = (int)(sh.off[d] + sh.cnt[w][d] + (pk & 0xffffu)), owner = pos / per, at = pos - owner * per;
      cl.map_shared_rank(dst, owner)[at] = pass ? src[e] : (unsigned)(i0 + e);
      cl.map_shared_rank(kdst, owner)[at] = ksrc[e];
    }
    cl.sync();
  }
  const int fb = (passes + 1) & 1;   // the buffers the last pass wrote: sh.idx[fb], sh.key[fb]
  // ---- voxel heads (first position of every run of equal keys) and their output indices; one contiguous chunk of positions per thread
  const int ch = (len + VGC_THREADS - 1) / VGC_THREADS, e0 = min(len, tid * ch), e1 = min(len, e0 + ch), g0 = c * per;
  unsigned prev = 0xffffffffu;   // no kept point has this key
  if (e0 < e1) prev = e0 ? sh.key[fb][e0 - 1] : c ? cl.map_shared_rank(sh.key[fb], c - 1)[per - 1] : 0xffffffffu;   // CTA c - 1 holds per positions
  unsigned nh = 0, p = prev;
#pragma unroll 1
  for (int e = e0; e < e1; e++) { const unsigned k = sh.key[fb][e]; nh += k != p; p = k; }
  unsigned cta_heads;
  const unsigned j0 = vgc_scan(sh, nh, &cta_heads);
  if (tid == 0) sh.n_heads = cta_heads;
  cl.sync();
  if (w == 0) {
    const unsigned h = lane < VGC_CTAS ? *cl.map_shared_rank(&sh.n_heads, lane) : 0u;
    const unsigned vbase = __reduce_add_sync(FULL, lane < c ? h : 0u), total = __reduce_add_sync(FULL, h);
    if (lane == 0) { sh.vbase = (int)vbase; sh.total = (int)total; if (c == 0) *sh.d_n_out = (int)total; }
  }
  __syncthreads();
  // ---- centroids: each thread sums the voxels whose head lies in its chunk, walking positions in ascending order (= ascending input index: the
  // sort is stable) with a sequential fp32 sum; the points of the chunk are loaded ahead, a voxel that runs past the chunk continues beyond it
  int o = sh.vbase + (int)j0;   // output index of the next voxel
  float sx = 0.f, sy = 0.f, sz = 0.f, si = 0.f; int cnt = 0; bool open = false;
  p = prev;
#pragma unroll 1
  for (int e = e0; e < e1; e += 4) {
    float4 pt[4];
#pragma unroll
    for (int u = 0; u < 4; u++) if (e + u < e1) pt[u] = __ldcg(in + sh.idx[fb][e + u]);
#pragma unroll
    for (int u = 0; u < 4; u++) {
      if (e + u >= e1) break;
      const unsigned k = sh.key[fb][e + u];
      if (k != p) {   // a head: close the open voxel, open this one
        if (open) { const float f = (float)cnt; sh.out[o++] = make_float4(sx / f, sy / f, sz / f, si / f); }
        sx = sy = sz = si = 0.f; cnt = 0; open = true; p = k;
      }
      if (open) { sx += pt[u].x; sy += pt[u].y; sz += pt[u].z; si += pt[u].w; cnt++; }
    }
  }
  if (open) {   // the last voxel opened in the chunk: its points past the chunk (a dense voxel holds a hundred points and more), four at a time
    const int nv = sh.g_n;
    bool done = false;
#pragma unroll 1
    for (int q = g0 + e1; q < nv;) {
      const int owner = q / per, qe = min(nv, (owner + 1) * per);
      const unsigned* kr = cl.map_shared_rank(sh.key[fb], owner) - owner * per;
      const unsigned* ir = cl.map_shared_rank(sh.idx[fb], owner) - owner * per;
#pragma unroll 1
      for (; q < qe; q += 4) {
        int m = 0;   // leading positions of the batch still in the voxel
#pragma unroll
        for (int u = 0; u < 4; u++) m += (m == u) & (q + u < qe && kr[q + u] == p);
#pragma unroll
        for (int h = 0; h < 4; h += 2) {
          float4 pt[2];
#pragma unroll
          for (int u = 0; u < 2; u++) if (h + u < m) pt[u] = __ldcg(in + ir[q + h + u]);
#pragma unroll
          for (int u = 0; u < 2; u++) if (h + u < m) { sx += pt[u].x; sy += pt[u].y; sz += pt[u].z; si += pt[u].w; cnt++; }
        }
        done = m < 4 && q + m < qe;   // a position of this CTA has another key
        if (done) break;
      }
      if (done) break;
      q = qe;
    }
    const float f = (float)cnt;
    sh.out[o] = make_float4(sx / f, sy / f, sz / f, si / f);
  }
  const int total = sh.total;
  cl.sync();
  return total;
}
struct VgClusterArgs { VgChainDev chain[2]; };
// Cluster k runs chain k.  64 registers and under 190 KB of shared memory per CTA: a solver CTA (256 threads x 128 registers) still fits
// on every SM that holds one.
__global__ void __maxnreg__(64) vg_cluster_chain_kernel(const VgClusterArgs a) {
  VgcShared& sh = *reinterpret_cast<VgcShared*>(vgc_smem);
  if (threadIdx.x == 0) sh.chain = blockIdx.x < VGC_CTAS ? a.chain[0] : a.chain[1];
  __syncthreads();
  int n = sh.chain.n_cap;
  if (sh.chain.d_n_in) n = max(0, min(*sh.chain.d_n_in, n));
  n = vgc_voxel_grid(0, n);
  if (sh.chain.nvg > 1) vgc_voxel_grid(1, n);
}
int voxel_grid_prepare(ll_ctx* ctx) {
  LL_CUDA(ctx, cudaFuncSetAttribute(vg_cluster_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(VgcShared)));
  LL_CUDA(ctx, cudaFuncSetAttribute(vg_cluster_chain_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));   // VGC_CTAS = 16
  return LL_OK;
}

// The one place that chooses how VoxelGrid chains run: every chain's host-known count within VG_CLUSTER_CAP -> one cluster launch of all the
// chains on s; else the CUB pass per VoxelGrid, each chain on its own stream (a chain on another stream than s forks from s through `fork`
// and s waits for it through `join`).
int launch_voxel_chains(ll_ctx* ctx, cudaStream_t s, const VgChain* c, int nchains, cudaEvent_t fork, cudaEvent_t join) {
  int n_max = 0;
  for (int k = 0; k < nchains; k++) n_max = std::max(n_max, c[k].d.n_cap);
  if (n_max <= VG_CLUSTER_CAP) {
    VgClusterArgs a = {};
    for (int k = 0; k < nchains; k++) a.chain[k] = c[k].d;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = VGC_CTAS; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(VGC_CTAS * nchains); cfg.blockDim = dim3(VGC_THREADS); cfg.dynamicSmemBytes = sizeof(VgcShared); cfg.stream = s;
    cfg.attrs = at; cfg.numAttrs = 1;
    LL_CUDA(ctx, cudaLaunchKernelEx(&cfg, vg_cluster_chain_kernel, a)); ctx->launches++;
    return LL_OK;
  }
  bool forked = false;
  for (int k = 0; k < nchains; k++) {
    const VgChain& ch = c[k];
    if (ch.s != s && !forked) { LL_CUDA(ctx, cudaEventRecord(fork, s)); forked = true; }
    if (ch.s != s) LL_CUDA(ctx, cudaStreamWaitEvent(ch.s, fork, 0));
    const float4* in = ch.d.in; const int* d_n = ch.d.d_n_in;
    for (int v = 0; v < ch.d.nvg; v++) {
      LL_TRY(launch_voxel_grid_segments(ctx, ch.s, *ch.scratch, in, ch.d.n_cap, d_n, 1, ch.d.leaf[v], ch.d.out[v], ch.d.d_n_out[v]));
      in = ch.d.out[v]; d_n = ch.d.d_n_out[v];
    }
    if (ch.s != s) LL_CUDA(ctx, cudaEventRecord(join, ch.s));
  }
  if (forked) LL_CUDA(ctx, cudaStreamWaitEvent(s, join, 0));
  return LL_OK;
}
int launch_voxel_grid(ll_ctx* ctx, cudaStream_t s, DevBuf& scratch, const float4* d_in, int n_cap, const int* d_n_in, float leaf, float4* d_out, int* d_n_out) {
  const VgChain c{{d_in, n_cap, d_n_in, 1, {leaf, 0.f}, {d_out, nullptr}, {d_n_out, nullptr}}, &scratch, s};
  return launch_voxel_chains(ctx, s, &c, 1, nullptr, nullptr);
}
