// Cloud plumbing kernels: format repack, pointAssociateToMap over a cloud, VoxelGrid down-sampling.
//
// Replaces, on the reference side:
//   pcl::VoxelGrid<PointXYZI>::filter (third-party PCL, restated)  call sites loam_livox/source/laser_feature_extractor.hpp:372-380,
//                                   loam_livox/source/laser_mapping.hpp:491,509,533-537,1367-1373,1434-1437                 (K4)
//   pointcloudAssociateToMap        loam_livox/source/point_cloud_registration.hpp:622-661,673-685                           (K6, cloud form)
//
// Compiled with -fmad=false (voxel indices, centroids and the transform must round like the scalar CPU code).
#include <cub/cub.cuh>
#include "common.cuh"
#include "kernels.cuh"
#include "exact_math.cuh"

#define FULL 0xffffffffu

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
  m->n_in = n - b; m->begin = b; m->passthrough = 0; m->ticket = 0;
  const float inv = 1.0f / leaf; m->inv = inv;
  if (v->n_finite == 0) { for (int k = 0; k < 3; k++) { m->min_b[k] = 0; m->mul[k] = 0; } return; }
  float mn[3], mx[3]; for (int k = 0; k < 3; k++) { mn[k] = key2f(~(unsigned)v->mn[k]); mx[k] = key2f((unsigned)v->mx[k]); }
  long long dx = (long long)((mx[0] - mn[0]) * inv) + 1, dy = (long long)((mx[1] - mn[1]) * inv) + 1, dz = (long long)((mx[2] - mn[2]) * inv) + 1;
  if (dx * dy * dz > 2147483647LL) { m->passthrough = 1; return; }
  int div_b[3];
  for (int k = 0; k < 3; k++) { m->min_b[k] = (int)floorf(mn[k] * inv); int max_b = (int)floorf(mx[k] * inv); div_b[k] = max_b - m->min_b[k] + 1; }
  m->mul[0] = 1; m->mul[1] = div_b[0]; m->mul[2] = div_b[0] * div_b[1];
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
    float4 p = in[i];
    if (m->passthrough) key = (unsigned)(i - m->begin);
    else if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
      const float inv = m->inv;
      int ijk0 = (int)(floorf(p.x * inv) - (float)m->min_b[0]);
      int ijk1 = (int)(floorf(p.y * inv) - (float)m->min_b[1]);
      int ijk2 = (int)(floorf(p.z * inv) - (float)m->min_b[2]);
      key = (unsigned)(ijk0 * m->mul[0] + ijk1 * m->mul[1] + ijk2 * m->mul[2]);
    }
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
int launch_voxel_grid(ll_ctx* ctx, cudaStream_t s, DevBuf& scratch, const float4* d_in, int n_cap, const int* d_n_in, float leaf, float4* d_out, int* d_n_out) {
  return launch_voxel_grid_segments(ctx, s, scratch, d_in, n_cap, d_n_in, 1, leaf, d_out, d_n_out);
}
