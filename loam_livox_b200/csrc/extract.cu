// Livox feature extraction kernels (K1 - K3).
//
// Replaces, on the reference side:
//   Livox_laser::projection_scan_3d_2d (+ eval_point, add_mask_of_point)   loam_livox/source/livox_feature_extractor.hpp:458-607,343-358,322-341   (K1)
//   Livox_laser::compute_features                                          loam_livox/source/livox_feature_extractor.hpp:361-455                    (K2)
//   Livox_laser::split_laser_scan (petal bookkeeping), piece bounds        loam_livox/source/livox_feature_extractor.hpp:657-719,
//                                                                          loam_livox/source/laser_feature_extractor.hpp:313-323
//   Livox_laser::get_features                                              loam_livox/source/livox_feature_extractor.hpp:219-272                    (K3)
//
// The reference walks the scan sequentially; here every per-point quantity is computed independently (the only true
// sequential dependences - "copy the previous point's projection for a zero return" and the 50-point split hysteresis -
// are a short walk-back per zero return and a single-thread pass over the few direction-flip candidates).
// Compiled with -fmad=false: all float arithmetic must round like the scalar CPU code.
#include <cub/cub.cuh>
#include "common.cuh"
#include "kernels.cuh"

#define SELF_EDGE_SRC 0x80   // private: this point raised e_pt_circle_edge (marks idx-2, idx-1, idx+1 too)
#define SELF_PROCESSED 0x40  // private: the point went through the normal projection path (e_pt_small_view_angle is never set by the reference)
#define PUBLIC_MASK 0x3f

struct ExtractParams {
  int n; float dt; const double* d_current_time;   // device scalar: the value changes per scan, the captured launch does not
  float min_dis_sq, min_sigma, max_edge_polar, thr_corner, thr_surface, min_view_angle;
};

__device__ __forceinline__ bool pt_is_nan(const float4& p) { return !isfinite(p.x) || !isfinite(p.y) || !isfinite(p.z); }

// pt_2d_img / polar_dis_sq2 of point j with the "x == 0 copies idx-1" rule resolved by walking back.
__device__ __forceinline__ void projection_of(const float4* __restrict__ raw, int j, float& u, float& v, float& polar) {
  for (;;) {
    const float4 p = raw[j];
    if (pt_is_nan(p)) { u = 0.f; v = 0.f; polar = 0.f; return; }        // Pt_infos defaults (pt_2d_img is uninitialised in the reference)
    if (p.x == 0.f && j > 0) { j--; continue; }
    u = p.y / p.x; v = p.z / p.x; polar = u * u + v * v; return;
  }
}

__global__ void ex_point_kernel(const float4* __restrict__ raw, ExtractParams P, float* __restrict__ time_stamp, float* __restrict__ polar_out, float* __restrict__ depth_out,
                                unsigned char* __restrict__ self_out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= P.n) return;
  const float4 p = raw[idx];
  time_stamp[idx] = (float)(*P.d_current_time + (double)(((float)idx) * P.dt));
  unsigned self = 0; float polar = 0.f, depth = 0.f;
  if (pt_is_nan(p)) self = LL_PT_NAN;
  else if (p.x == 0.f && idx > 0) { self = LL_PT_000; float u, v; projection_of(raw, idx - 1, u, v, polar); }
  else {
    if (p.x == 0.f) self |= LL_PT_000;   // first point of the scan: masked but still projected (:495-504)
    depth = p.x * p.x + p.y * p.y + p.z * p.z;
    const float u = p.y / p.x, v = p.z / p.x; polar = u * u + v * v;
    if (depth < P.min_dis_sq) self |= LL_PT_TOO_NEAR;
    const float sigma = p.w / polar;
    if (sigma < P.min_sigma) self |= LL_PT_REFLECTIVITY_LOW;
    if (polar > P.max_edge_polar) self |= LL_PT_CIRCLE_EDGE | SELF_EDGE_SRC;
    self |= SELF_PROCESSED;
  }
  polar_out[idx] = polar; depth_out[idx] = depth; self_out[idx] = (unsigned char)self;
}

__device__ __forceinline__ int dir_of(const float* __restrict__ polar, const unsigned char* __restrict__ self, int j) {
  if (j < 1 || !(self[j] & SELF_PROCESSED)) return 0;
  const float d = polar[j] - polar[j - 1];
  return d > 0.f ? 1 : (d < 0.f ? -1 : 0);
}

__global__ void ex_feature_kernel(const float4* __restrict__ raw, ExtractParams P, const float* __restrict__ polar, const float* __restrict__ depth, const unsigned char* __restrict__ self,
                                  int* __restrict__ pt_type, int* __restrict__ pt_label, float* __restrict__ curvature, float* __restrict__ view_angle,
                                  signed char* __restrict__ polar_dir, unsigned char* __restrict__ cand) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x, n = P.n;
  if (idx >= n) return;
  const unsigned s0 = self[idx];
  unsigned type = s0 & PUBLIC_MASK;
  if ((idx + 1 < n && (self[idx + 1] & SELF_EDGE_SRC)) || (idx + 2 < n && (self[idx + 2] & SELF_EDGE_SRC)) || (idx >= 1 && (self[idx - 1] & SELF_EDGE_SRC))) type |= LL_PT_CIRCLE_EDGE;
  pt_type[idx] = (int)type;
  // petal split candidates (:529-562)
  const int dcur = dir_of(polar, self, idx);
  polar_dir[idx] = (signed char)dcur;
  unsigned char c = 0;
  if (idx >= 1 && (s0 & SELF_PROCESSED)) {
    const int dprev = dir_of(polar, self, idx - 1);
    if (dcur == -1 && dprev == 1) c = 1; else if (dcur == 1 && dprev == -1) c = 2;
  }
  cand[idx] = c;
  // curvature / view angle / labels (:361-455)
  int label = 0; float curv = 0.f, va = 0.f;
  if (idx >= 2 && idx < n - 2 && !(s0 & (LL_PT_000 | LL_PT_NAN))) {
    const float4 p = raw[idx];
    float ax = 0.f, ay = 0.f, az = 0.f;
#pragma unroll
    for (int i = 1; i <= 2; i++) {
      const unsigned tp = self[idx + i], tm = self[idx - i];
      if ((tp | tm) & LL_PT_000) { if (i == 1) label |= LL_LABEL_NEAR_ZERO; else label = LL_LABEL_INVALID; break; }
      else if ((tp | tm) & LL_PT_NAN) { if (i == 1) label |= LL_LABEL_NEAR_NAN; else label = LL_LABEL_INVALID; break; }
      else { const float4 a = raw[idx + i], b = raw[idx - i]; ax += a.x + b.x; ay += a.y + b.y; az += a.z + b.z; }
    }
    if (label != LL_LABEL_INVALID) {
      ax -= 4.0f * p.x; ay -= 4.0f * p.y; az -= 4.0f * p.z;
      curv = ax * ax + ay * ay + az * az;
      const float4 q2 = raw[idx + 2], q0 = raw[idx - 2];
      const float bx = q2.x - q0.x, by = q2.y - q0.y, bz = q2.z - q0.z;
      // Eigen_math::vector_angle(vec_a, vec_b, 1) * 57.3 ; Eigen's 3-vector reductions associate as x + (y + z)
      const float an = sqrtf(p.x * p.x + (p.y * p.y + p.z * p.z)), bn = sqrtf(bx * bx + (by * by + bz * bz));
      float ang = 0.f;
      if (!(an == 0.f || bn == 0.f)) { const float d = p.x * bx + (p.y * by + p.z * bz); ang = (float)acos((double)(fabsf(d) / (an * bn))); }
      va = (float)((double)ang * 57.3);
      if (va > P.min_view_angle) {
        if (curv < P.thr_surface) label |= LL_LABEL_SURFACE;
        if (curv > P.thr_corner) {
          const float d0 = depth[idx], dm = depth[idx - 2], dp = depth[idx + 2];
          if (d0 <= dm && d0 <= dp) { if (fabsf(d0 - dm) < 0.1f * d0 || fabsf(d0 - dp) < 0.1f * d0) label |= LL_LABEL_CORNER; }
        }
      }
    }
  }
  pt_label[idx] = label; curvature[idx] = curv; view_angle[idx] = va;
}

// Single warp: 50-point hysteresis over the flip candidates, petal angles, grouping, first / last surviving point per petal.
// meta: [0] n_split, [1] n_scans (petals handed to the caller), [2] clutter_size
__global__ void ex_petal_kernel(const float4* __restrict__ raw, int n, const float* __restrict__ polar, const int* __restrict__ pt_type, const unsigned char* __restrict__ cand,
                                const int* __restrict__ cand_idx, const int* __restrict__ d_num_cand, int* __restrict__ split, float* __restrict__ seg_angle,
                                int* __restrict__ scan_first, int* __restrict__ scan_last, int* __restrict__ meta) {
  const int lane = threadIdx.x;
  __shared__ int s_nsplit, s_ngroup;
  __shared__ int s_c[256];
  {
    // lane 0 walks the candidates in order (the hysteresis is sequential), the warp stages them through shared memory 256 at a time
    // so that the walk does not pay two dependent global loads per candidate.
    int ns = 0, n_edge = 0, n_zero = 0, last_split = 0; const int nc = *d_num_cand;
    for (int base = 0; base < nc; base += 256) {
      for (int k = lane; k < 256 && base + k < nc; k += 32) { const int idx = cand_idx[base + k]; s_c[k] = (idx << 2) | (int)cand[idx]; }
      __syncwarp();
      if (lane == 0) {
        const int m = min(256, nc - base);
        for (int k = 0; k < m; k++) {
          const int idx = s_c[k] >> 2, t = s_c[k] & 3;
          if (t == 1) { if (n_edge == 0 || (idx - last_split) > 50) { split[ns++] = idx; last_split = idx; n_edge++; } }
          else if (t == 2) { if (n_zero == 0 || (idx - last_split) > 50) { split[ns++] = idx; last_split = idx; n_zero++; } }
        }
      }
      __syncwarp();
    }
    if (lane == 0) {
      split[ns++] = n - 1;
      s_nsplit = ns; meta[0] = ns;
      if (ns < 6) { meta[1] = 0; meta[2] = 0; } else meta[2] = ns - 1;
    }
  }
  __syncwarp();
  const int ns = s_nsplit;
  if (ns < 6) return;
  const int nseg = ns - 1;
  for (int k = lane; k < nseg; k += 32) {
    const int internal = split[k + 1] - split[k];
    int pidx;
    if (polar[split[k + 1]] > 10000.f) pidx = split[k + 1] - (int)(internal * 0.20); else pidx = split[k + 1] - (int)(internal * 0.80);
    float u, v, pl; projection_of(raw, pidx, u, v, pl);
    float ang = (float)(atan2((double)v, (double)u) * 57.3);
    seg_angle[k] = (float)(ang + 180.0);
  }
  __syncwarp();
  // group consecutive segments with identical angle (scan_id_index changes), drop the last group (laserCloudScans.resize(scan_idx)),
  // keep groups with at least one surviving point.  Group boundaries are written into scan_first/scan_last temporarily.
  if (lane == 0) {
    int g = 0;
    for (int k = 0; k < nseg; k++) {
      const int b = (k == 0) ? 0 : split[k] + 1, e = split[k + 1];
      if (k > 0 && seg_angle[k] == seg_angle[k - 1]) { scan_last[g - 1] = e; }
      else { if (e >= b || k == 0) { scan_first[g] = b; scan_last[g] = e; g++; } }
    }
    s_ngroup = g - 1;   // last one dropped
  }
  __syncwarp();
  const int ng = s_ngroup;
  const int remove_type = LL_PT_000 | LL_PT_TOO_NEAR | LL_PT_NAN;
  for (int g = lane; g < ng; g += 32) {
    const int b = scan_first[g], e = scan_last[g]; int first = -1, last = -1;
    for (int i = b; i <= e; i++) if ((pt_type[i] & remove_type) == 0 && raw[i].x != 0.f) { first = i; break; }
    if (first >= 0) for (int i = e; i >= b; i--) if ((pt_type[i] & remove_type) == 0 && raw[i].x != 0.f) { last = i; break; }
    scan_first[g] = first; scan_last[g] = last;
  }
  __syncwarp();
  if (lane == 0) {
    int m = 0;
    for (int g = 0; g < ng; g++) if (scan_first[g] >= 0) { scan_first[m] = scan_first[g]; scan_last[m] = scan_last[g]; m++; }
    meta[1] = m;
  }
}

// laser_feature_extractor.hpp:313-323 ; out[2*i] = start, out[2*i+1] = end
__global__ void ex_piece_kernel(const int* __restrict__ scan_first, const int* __restrict__ scan_last, const int* __restrict__ meta, int n, int pieces, float* __restrict__ out) {
  const int i = threadIdx.x; if (i >= pieces) return;
  const int nscan = meta[1];
  if (nscan <= 0) { out[2 * i] = 0.f; out[2 * i + 1] = 0.f; return; }
  const int start_scans = (nscan * i) / pieces, end_scans = (nscan * (i + 1)) / pieces - 1;
  out[2 * i] = ((float)scan_first[start_scans]) / (float)n;
  out[2 * i + 1] = ((float)scan_last[end_scans < 0 ? 0 : end_scans]) / (float)n;
}

// K3: membership flags packed for one 64-bit prefix sum: bits 0-20 corner, 21-41 surface, 42-62 full
__global__ void ex_flags_kernel(int n, const int* __restrict__ pt_type, const int* __restrict__ pt_label, const float* __restrict__ depth, const float* __restrict__ d_bounds,
                                float min_blur, float max_blur, unsigned long long* __restrict__ packed, int* __restrict__ counts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) { counts[10] = ll_f2ord(10000.0f); counts[11] = ll_f2ord(-10000.0f); }   // find_min_max_intensity's start values (laser_mapping.hpp:1246-1247)
  if (i >= n) return;
  if (d_bounds) { min_blur = d_bounds[0]; max_blur = d_bounds[1]; }
  const float maximum_idx = max_blur * (float)n, minimum_idx = min_blur * (float)n;
  unsigned long long f = 0;
  const float fi = (float)i;
  if (!(fi > maximum_idx || fi < minimum_idx)) {
    const int type = pt_type[i], label = pt_label[i]; bool skip_full = false;
    if ((type & (LL_PT_000 | LL_PT_NAN | LL_PT_TOO_NEAR)) == 0) {
      if (label & LL_LABEL_CORNER) {
        if (type != LL_PT_NORMAL) skip_full = true;   // the early `continue` (:240-241) also skips the surface test and the full cloud
        else if ((double)depth[i] < 900.0) f |= 1ull;
      }
      if (!skip_full && (label & LL_LABEL_SURFACE)) { if ((double)depth[i] < 1000000.0) f |= 1ull << 21; }
    }
    if (!skip_full) f |= 1ull << 42;
  }
  packed[i] = f;
}
__global__ void ex_scatter_kernel(int n, const float4* __restrict__ raw, const float* __restrict__ time_stamp, const unsigned long long* __restrict__ packed,
                                  const unsigned long long* __restrict__ offs, float4* __restrict__ corners, float4* __restrict__ surf, float4* __restrict__ full, int* __restrict__ counts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = i < n;
  const unsigned long long f = in ? packed[i] : 0ull, o = in ? offs[i] : 0ull;
  float4 p = make_float4(0.f, 0.f, 0.f, 0.f); if (in) { p = raw[i]; p.w = time_stamp[i]; }
  // find_min_max_intensity over the full cloud (laser_mapping.hpp:1243-1253, :1336): min / max time stamp of the points that go to `full`
  { const bool fl = (f >> 42) & 1ull; const int k = ll_f2ord(p.w);
    const int mn = __reduce_min_sync(0xffffffffu, fl ? k : 0x7fffffff), mx = __reduce_max_sync(0xffffffffu, fl ? k : (int)0x80000000);
    if ((threadIdx.x & 31) == 0 && mn != 0x7fffffff) { atomicMin(&counts[10], mn); atomicMax(&counts[11], mx); } }
  if (!in) return;
  if (f & 1ull) corners[(int)(o & 0x1fffff)] = p;
  if (f & (1ull << 21)) surf[(int)((o >> 21) & 0x1fffff)] = p;
  if ((f & (1ull << 42)) && full) full[(int)((o >> 42) & 0x1fffff)] = p;
  if (i == n - 1) { const unsigned long long t = o + f; counts[0] = (int)(t & 0x1fffff); counts[1] = (int)((t >> 21) & 0x1fffff); counts[2] = (int)((t >> 42) & 0x1fffff); }
}

// ------------------------------------------------------------------------------------------------ host side
int extract_alloc(ll_ctx* ctx) {
  ExtractState& e = ctx->ex;
  const size_t n = (size_t)ctx->cfg.max_scan_points;
  LL_CUDA(ctx, ctx->extract_buf.carve([&](Carve& c) {
    e.raw = c.take<float4>(n);
    e.pt_type = c.take<int>(n); e.pt_label = c.take<int>(n);
    e.curvature = c.take<float>(n); e.view_angle = c.take<float>(n); e.depth_sq2 = c.take<float>(n);
    e.time_stamp = c.take<float>(n); e.polar_dis_sq2 = c.take<float>(n);
    e.polar_dir = c.take<int8_t>(n); e.self_mask = c.take<uint8_t>(n); e.cand = c.take<uint8_t>(n);
    e.cand_idx = c.take<int>(n); e.split_idx = c.take<int>(n + 1);
    e.scan_first = c.take<int>(n + 1); e.scan_last = c.take<int>(n + 1);
    e.d_num_cand = c.take<int>(1); e.d_meta = c.take<int>(4); e.d_time = c.take<double>(1);
  }));
  return LL_OK;
}

static ExtractParams extract_params(ll_ctx* ctx, int n) {
  ExtractState& e = ctx->ex;
  ExtractParams P; P.n = n; P.dt = ctx->cfg.time_interval_pts; P.d_current_time = e.d_time;
  P.min_dis_sq = ctx->cfg.livox_min_dis * ctx->cfg.livox_min_dis; P.min_sigma = ctx->cfg.livox_min_sigma;
  P.max_edge_polar = (float)std::pow(std::tan(ctx->cfg.max_fov_deg / 57.3) * 1, 2);
  P.thr_corner = ctx->cfg.corner_curvature; P.thr_surface = ctx->cfg.surface_curvature; P.min_view_angle = ctx->cfg.minimum_view_angle;
  return P;
}
// K1 + K2: the per-point part of projection_scan_3d_2d and compute_features (everything get_features needs)
int launch_extract_points(ll_ctx* ctx, int n) {
  ExtractState& e = ctx->ex; cudaStream_t s = ctx->stream;
  const ExtractParams P = extract_params(ctx, n);
  const int blocks = ll_div_up(n, 256);
  ex_point_kernel<<<blocks, 256, 0, s>>>(e.raw, P, e.time_stamp, e.polar_dis_sq2, e.depth_sq2, e.self_mask);
  ex_feature_kernel<<<blocks, 256, 0, s>>>(e.raw, P, e.polar_dis_sq2, e.depth_sq2, e.self_mask, e.pt_type, e.pt_label, e.curvature, e.view_angle, (signed char*)e.polar_dir, e.cand);
  ctx->launches += 2;
  LL_CUDA(ctx, cudaGetLastError());
  return LL_OK;
}
// The petal bookkeeping (split indices with the 50-point hysteresis, petal angles, first / last surviving point per petal: :529-604, split_laser_scan).
// Only the piece bounds and the "<= 5 petals" test read its results, so with whole_frame = 1 the front end runs it on a side stream.
// CUB temp | petal angles
struct PetalsLayout {
  size_t sel_bytes = 0; char* tmp; float* seg_angle;
  explicit PetalsLayout(int n) { cub::DeviceSelect::Flagged(nullptr, sel_bytes, cub::CountingInputIterator<int>(0), (unsigned char*)nullptr, (int*)nullptr, (int*)nullptr, n); }
  void layout(Carve& c, int n) { tmp = c.take<char>(sel_bytes); seg_angle = c.take<float>(n + 1); }
};
size_t petals_bytes(int n) { PetalsLayout P(n); return layout_bytes([&](Carve& c) { P.layout(c, n); }); }
int launch_extract_petals(ll_ctx* ctx, int n, cudaStream_t s, DevBuf& scratch) {
  ExtractState& e = ctx->ex;
  PetalsLayout P(n);
  LL_CUDA(ctx, scratch.carve([&](Carve& c) { P.layout(c, n); }));
  LL_CUDA(ctx, cub::DeviceSelect::Flagged(P.tmp, P.sel_bytes, cub::CountingInputIterator<int>(0), e.cand, e.cand_idx, e.d_num_cand, n, s));
  ex_petal_kernel<<<1, 32, 0, s>>>(e.raw, n, e.polar_dis_sq2, e.pt_type, e.cand, e.cand_idx, e.d_num_cand, e.split_idx, P.seg_angle, e.scan_first, e.scan_last, e.d_meta);
  ctx->launches += 3;
  LL_CUDA(ctx, cudaGetLastError());
  return LL_OK;
}

int launch_piece_bounds(ll_ctx* ctx, int pieces, float* d_start_end) {
  ExtractState& e = ctx->ex;
  ex_piece_kernel<<<1, 32, 0, ctx->stream>>>(e.scan_first, e.scan_last, e.d_meta, e.n, pieces, d_start_end); ctx->launches++;
  LL_CUDA(ctx, cudaGetLastError());
  return LL_OK;
}

// flags | their prefix sum | CUB temp
struct FeaturesLayout {
  size_t scan_bytes = 0; unsigned long long* packed; unsigned long long* offs; char* tmp;
  explicit FeaturesLayout(int n) { cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (unsigned long long*)nullptr, (unsigned long long*)nullptr, n); }
  void layout(Carve& c, int n) { packed = c.take<unsigned long long>(n); offs = c.take<unsigned long long>(n); tmp = c.take<char>(scan_bytes); }
};
size_t get_features_bytes(int n) { FeaturesLayout F(n); return layout_bytes([&](Carve& c) { F.layout(c, n); }); }
int launch_get_features(ll_ctx* ctx, cudaStream_t s, DevBuf& scratch, const float* d_bounds, float min_blur, float max_blur, float4* d_corners, float4* d_surf, float4* d_full, int* d_counts) {
  ExtractState& e = ctx->ex; const int n = e.n;
  if (n == 0) { LL_CUDA(ctx, cudaMemsetAsync(d_counts, 0, 3 * sizeof(int), s)); return LL_OK; }
  FeaturesLayout F(n);
  LL_CUDA(ctx, scratch.carve([&](Carve& c) { F.layout(c, n); }));
  const int blocks = ll_div_up(n, 256);
  ex_flags_kernel<<<blocks, 256, 0, s>>>(n, e.pt_type, e.pt_label, e.depth_sq2, d_bounds, min_blur, max_blur, F.packed, d_counts);
  LL_CUDA(ctx, cub::DeviceScan::ExclusiveSum(F.tmp, F.scan_bytes, F.packed, F.offs, n, s));
  ex_scatter_kernel<<<blocks, 256, 0, s>>>(n, e.raw, e.time_stamp, F.packed, F.offs, d_corners, d_surf, d_full, d_counts);
  ctx->launches += 4;
  LL_CUDA(ctx, cudaGetLastError());
  return LL_OK;
}
