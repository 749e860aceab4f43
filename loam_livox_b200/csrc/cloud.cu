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

int upload_cloud(ll_ctx* ctx, const void* src, size_t n, int fmt, int where, float4* d_dst) {
  if (n == 0) return LL_OK;
  cudaStream_t s = ctx->stream;
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
struct VgMeta {
  int mn[3], mx[3];     // ordered-int encodings of the float min / max
  int n_finite;
  int passthrough;      // dx*dy*dz overflows int32: PCL warns and copies the input through
  int n_in;
  int min_b[3]; int mul[3];
  float inv;
  int ticket;           // blocks of vg_minmax_setup_kernel that have finished (the last one does the set-up and resets it)
};

// Min / max over the finite points, then -- by the last block to finish -- the grid set-up of VoxelGrid::applyFilter (one launch instead of
// init + minmax + setup; `m` is cleared by a memset node: mins are kept as the bitwise complement of their order-preserving key, so that
// "all zero" is the neutral element of the atomicMax that reduces both the mins and the maxs).
__device__ __forceinline__ unsigned f2key(float f) { return (unsigned)ll_f2ord(f) ^ 0x80000000u; }     // unsigned order == float order
__device__ __forceinline__ float key2f(unsigned k) { return ll_ord2f((int)(k ^ 0x80000000u)); }
__global__ void vg_minmax_setup_kernel(const float4* __restrict__ in, VgMeta* m, int n_host, const int* __restrict__ d_n, float leaf) {
  const int n = d_n ? min(*d_n, n_host) : n_host;
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY}; int cnt = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
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
  m->n_in = n; m->passthrough = 0; m->ticket = 0;
  const float inv = 1.0f / leaf; m->inv = inv;
  if (v->n_finite == 0) { for (int k = 0; k < 3; k++) { m->min_b[k] = 0; m->mul[k] = 0; } return; }
  float mn[3], mx[3]; for (int k = 0; k < 3; k++) { mn[k] = key2f(~(unsigned)v->mn[k]); mx[k] = key2f((unsigned)v->mx[k]); }
  long long dx = (long long)((mx[0] - mn[0]) * inv) + 1, dy = (long long)((mx[1] - mn[1]) * inv) + 1, dz = (long long)((mx[2] - mn[2]) * inv) + 1;
  if (dx * dy * dz > 2147483647LL) { m->passthrough = 1; return; }
  int div_b[3];
  for (int k = 0; k < 3; k++) { m->min_b[k] = (int)floorf(mn[k] * inv); int max_b = (int)floorf(mx[k] * inv); div_b[k] = max_b - m->min_b[k] + 1; }
  m->mul[0] = 1; m->mul[1] = div_b[0]; m->mul[2] = div_b[0] * div_b[1];
}
__global__ void vg_keys_kernel(const float4* __restrict__ in, const VgMeta* __restrict__ m, int n_cap, unsigned* __restrict__ keys, int* __restrict__ vals) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_cap) return;
  unsigned key = 0xffffffffu;
  if (i < m->n_in) {
    float4 p = in[i];
    if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
      const float inv = m->inv;
      int ijk0 = (int)(floorf(p.x * inv) - (float)m->min_b[0]);
      int ijk1 = (int)(floorf(p.y * inv) - (float)m->min_b[1]);
      int ijk2 = (int)(floorf(p.z * inv) - (float)m->min_b[2]);
      key = (unsigned)(ijk0 * m->mul[0] + ijk1 * m->mul[1] + ijk2 * m->mul[2]);
    }
  }
  keys[i] = key; vals[i] = i;
}
// First element of every run of equal (valid) keys in the sorted key array: the predicate of the stream compaction that lists the voxels.
struct VgHead {
  const unsigned* keys;
  __device__ __forceinline__ bool operator()(int i) const { const unsigned k = keys[i]; return k != 0xffffffffu && (i == 0 || keys[i - 1] != k); }
};
// One thread per voxel: sequential float sum in ascending input index (radix sort is stable), like CentroidPoint<PointXYZI>.
__global__ void vg_centroid_kernel(const float4* __restrict__ in, const VgMeta* __restrict__ m, const int* __restrict__ vals, const int* __restrict__ seg_start,
                                   const int* __restrict__ d_num_seg, int n_cap, float4* __restrict__ out, int* __restrict__ d_n_out) {
  int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (m->passthrough) {
    if (s < m->n_in) out[s] = in[s];
    if (s == 0) *d_n_out = m->n_in;
    return;
  }
  const int nseg = *d_num_seg;
  if (s == 0) *d_n_out = nseg;
  if (s >= nseg) return;
  const int b = seg_start[s], e = (s + 1 < nseg) ? seg_start[s + 1] : m->n_finite;
  float sx = 0.f, sy = 0.f, sz = 0.f, si = 0.f;
  for (int li = b; li < e; li++) { const float4 p = in[vals[li]]; sx += p.x; sy += p.y; sz += p.z; si += p.w; }
  const float cnt = (float)(e - b);
  out[s] = make_float4(sx / cnt, sy / cnt, sz / cnt, si / cnt);
}

// The scratch of one VoxelGrid over n_cap points (n_cap > 0).
struct VgScratch {
  size_t sort_bytes = 0, sel_bytes = 0;
  VgMeta* meta; int* d_num_seg; unsigned* k0; unsigned* k1; int* v0; int* v1; int* seg; char* tmp;
  explicit VgScratch(int n_cap) {
    cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (unsigned*)nullptr, (unsigned*)nullptr, (int*)nullptr, (int*)nullptr, n_cap, 0, 32);
    cub::DeviceSelect::If(nullptr, sel_bytes, cub::CountingInputIterator<int>(0), (int*)nullptr, (int*)nullptr, n_cap, VgHead{nullptr});
  }
  void layout(Carve& c, int n_cap) {
    meta = c.take<VgMeta>(1); d_num_seg = c.take<int>(1);
    k0 = c.take<unsigned>(n_cap); k1 = c.take<unsigned>(n_cap); v0 = c.take<int>(n_cap); v1 = c.take<int>(n_cap); seg = c.take<int>(n_cap);
    tmp = c.take<char>(sort_bytes > sel_bytes ? sort_bytes : sel_bytes);
  }
};
size_t voxel_grid_bytes(int n_cap) {
  if (n_cap <= 0) return 0;
  VgScratch v(n_cap);
  return layout_bytes([&](Carve& c) { v.layout(c, n_cap); });
}
// On an explicit stream with its own scratch arena: VoxelGrid chains run side by side (every kernel here is far too small to fill the GPU,
// so the chains overlap almost perfectly).
int launch_voxel_grid(ll_ctx* ctx, cudaStream_t s, DevBuf& scratch, const float4* d_in, int n_cap, const int* d_n_in, float leaf, float4* d_out, int* d_n_out) {
  if (n_cap <= 0) { LL_CUDA(ctx, cudaMemsetAsync(d_n_out, 0, sizeof(int), s)); return LL_OK; }
  VgScratch v(n_cap);
  LL_CUDA(ctx, scratch.carve([&](Carve& c) { v.layout(c, n_cap); }));
  const int blocks = ll_div_up(n_cap, 256);
  LL_CUDA(ctx, cudaMemsetAsync(v.meta, 0, sizeof(VgMeta), s));
  vg_minmax_setup_kernel<<<min(blocks, ctx->num_sms * 2), 256, 0, s>>>(d_in, v.meta, n_cap, d_n_in, leaf);
  vg_keys_kernel<<<blocks, 256, 0, s>>>(d_in, v.meta, n_cap, v.k0, v.v0);
  LL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(v.tmp, v.sort_bytes, v.k0, v.k1, v.v0, v.v1, n_cap, 0, 32, s));
  LL_CUDA(ctx, cub::DeviceSelect::If(v.tmp, v.sel_bytes, cub::CountingInputIterator<int>(0), v.seg, v.d_num_seg, n_cap, VgHead{v.k1}, s));
  vg_centroid_kernel<<<blocks, 256, 0, s>>>(d_in, v.meta, v.v1, v.seg, v.d_num_seg, n_cap, d_out, d_n_out);
  ctx->launches += 11;   // minmax+setup, keys, radix sort (histogram, scan, 4 onesweep passes), select (init, sweep), centroid
  LL_CUDA(ctx, cudaGetLastError());
  return LL_OK;
}
