// Relocalization (include/loamlivox_b200.h, ll_reloc_*; DESIGN.md §4.3): the pose of a scan in a prior map without an initial guess.
// An occupancy bitmask of the map's own device clouds, dilated; every hypothesis of a rotation set x translation lattice scored by how many
// score points land on set voxels; the first K local maxima (peaks) of the score field refined by the batched registration (ll_register_batch).
// Beyond the reference, which has no relocalization: its only answer to a lost track is to drop the scan (laser_mapping.hpp:1413-1416).
//
// Built -fmad=false: the cell of a point and the transform of a score point are restated bit for bit by tests/reloc_reference.py
// (the occupancy index) and tests/reloc_field_reference.py (the distance fields).
#include <cmath>
#include <algorithm>
#include "common.cuh"
#include "kernels.cuh"
#include "exact_math.cuh"
#include <math_constants.h>

#define RELOC_MAX_DILATE 4
#define RELOC_MAX_HYP (1 << 24)
#define RELOC_MAX_VOXELS (1ll << 30)
#define RELOC_TILE 1024    // score points rotated into shared memory per pass (3 x 8 KB)
#define RELOC_GROUP 64     // lattice translations per CTA (8 warps x 8)

namespace {
struct RelocGrid { const uint32_t* bits; int dims[3]; double lo[3]; double res; int dilate; };

// What both searches keep: the map a search was built on, its grid and the buffers of its coarse stage.
struct RelocBase {
  int device = 0;
  const ll_map* map = nullptr; const float4* src[2] = {nullptr, nullptr}; int n_src[2] = {0, 0};   // the map it was built on
  RelocGrid grid = {};   // dilate: the index's dilate, the field's trunc; bits: the index's bitmask, null for the field
  int max_hyp = 0;
  long long n_vox = 0;
  DevBuf storage;   // everything below and the derived object's arrays, allocated once by its build
  int32_t* scores = nullptr;            // [max_hyp] coarse scores
  unsigned long long* peaks = nullptr;  // [max_hyp] peak keys (score << 32 | ~h), unordered
  int* counts = nullptr;                // [0] peaks, [1] candidates
  unsigned long long* cand = nullptr;   // [LL_MAX_BATCH] the first K peaks
};
}  // namespace

struct ll_reloc_index : RelocBase {
  long long n_words = 0;
  uint32_t* bits = nullptr;             // [n_words] the dilated occupancy, x fastest, bit v & 31 of word v >> 5
  float4* pts = nullptr;                // [LL_RELOC_MAX_SCORE_POINTS] score points (scan frame)
  double* rot = nullptr;                // [max_hyp x 4] hypothesis rotations (w, x, y, z)
};

#define RELOC_MAX_TRUNC 15   // T^2 <= 225 fits a byte

struct ll_reloc_field : RelocBase {
  uint8_t* d2[2] = {nullptr, nullptr};  // [n_vox] per class ([0] corner, [1] surface): min(T^2, squared voxel distance to the class's nearest point)
  int32_t* fine = nullptr;              // [max_hyp] the fine groups' scores, group-major
  unsigned long long* picks = nullptr;  // [LL_MAX_BATCH] each fine group's pick key (score << 32 | ~index)
  int32_t* verify = nullptr;            // [LL_MAX_BATCH] the score of each refined pose
  float4* pts[2] = {nullptr, nullptr};  // [LL_RELOC_MAX_SCORE_POINTS] score points per class (scan frame)
  double* rot = nullptr;                // [max_hyp x 4] the rotations of every group, group-major
  double* t0 = nullptr;                 // [LL_MAX_BATCH x 3] each group's lattice origin
};

namespace {

// Cell of p on axis a = floor((p_a - lo_a) / res) + dilate in fp64, compared as a double before it becomes an integer.
__device__ __forceinline__ bool grid_cell(const RelocGrid& g, float x, float y, float z, long long* v) {
  const float p[3] = {x, y, z};
  long long c[3];
  for (int a = 0; a < 3; a++) {
    const double d = floor(((double)p[a] - g.lo[a]) / g.res) + (double)g.dilate;
    if (!(d >= 0.0 && d < (double)g.dims[a])) return false;
    c[a] = (long long)d;
  }
  *v = c[0] + (long long)g.dims[0] * (c[1] + (long long)g.dims[1] * c[2]);
  return true;
}

__global__ void reloc_mark_kernel(const float4* __restrict__ src, int n, RelocGrid g, uint32_t* __restrict__ bits) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 p = src[i];
  if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) return;
  long long v;
  if (grid_cell(g, p.x, p.y, p.z, &v)) atomicOr(&bits[v >> 5], 1u << (v & 31));
}

// One separable pass of the Chebyshev dilation along `axis` (radius r, clipped at the border): one thread per voxel, one ballot per word.
__global__ void reloc_dilate_kernel(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, int d0, int d1, int d2, int axis, int r, long long n_vox,
                                    long long n_words) {
  const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  bool set = false;
  if (v < n_vox) {
    const long long yz = v / d0;
    const int x = (int)(v - yz * d0), y = (int)(yz % d1), z = (int)(yz / d1);
    const int c = axis == 0 ? x : (axis == 1 ? y : z), D = axis == 0 ? d0 : (axis == 1 ? d1 : d2);
    const long long stride = axis == 0 ? 1 : (axis == 1 ? (long long)d0 : (long long)d0 * d1);
    const int a = max(c - r, 0), b = min(c + r, D - 1);
    for (int k = a; k <= b && !set; k++) { const long long u = v + (long long)(k - c) * stride; set = (in[u >> 5] >> (u & 31)) & 1u; }
  }
  const unsigned w = __ballot_sync(0xffffffffu, set);
  if ((threadIdx.x & 31) == 0 && (v >> 5) < n_words) out[v >> 5] = w;
}

struct ScoreArgs {
  RelocGrid g; const float4* pts; int n_pts; const double* rot;
  double t0[3], step[3]; int nt[3]; int n_lat, blocks_per_rot;
  int32_t* scores;
};
// CTA = one rotation x RELOC_GROUP consecutive lattice points.  Per tile, the score points are rotated once (qrot_d, fp64) into shared memory;
// then one warp per translation counts, its lanes striding over the tile.  score(h) with h = l + n_lat * r, l = i + nt0 (j + nt1 k).
__global__ void __launch_bounds__(256) reloc_score_kernel(ScoreArgs a) {
  __shared__ double sx[RELOC_TILE], sy[RELOC_TILE], sz[RELOC_TILE];
  __shared__ int cnt[RELOC_GROUP];
  const int r = blockIdx.x / a.blocks_per_rot, l0 = (blockIdx.x - r * a.blocks_per_rot) * RELOC_GROUP;
  const double q[4] = {a.rot[4 * r], a.rot[4 * r + 1], a.rot[4 * r + 2], a.rot[4 * r + 3]};
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, n_warps = blockDim.x >> 5;
  if (threadIdx.x < RELOC_GROUP) cnt[threadIdx.x] = 0;
  for (int base = 0; base < a.n_pts; base += RELOC_TILE) {
    const int nt = min(RELOC_TILE, a.n_pts - base);
    __syncthreads();
    for (int i = threadIdx.x; i < nt; i += blockDim.x) {
      const float4 p = a.pts[base + i];
      double ox = CUDART_NAN, oy = CUDART_NAN, oz = CUDART_NAN;   // a point with a non-finite coordinate never scores
      if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) qrot_d(q, (double)p.x, (double)p.y, (double)p.z, ox, oy, oz);
      sx[i] = ox; sy[i] = oy; sz[i] = oz;
    }
    __syncthreads();
    for (int j = warp; j < RELOC_GROUP; j += n_warps) {
      const int l = l0 + j;
      if (l >= a.n_lat) break;
      const int i0 = l % a.nt[0], i1 = (l / a.nt[0]) % a.nt[1], i2 = l / (a.nt[0] * a.nt[1]);
      const double tx = a.t0[0] + (double)i0 * a.step[0], ty = a.t0[1] + (double)i1 * a.step[1], tz = a.t0[2] + (double)i2 * a.step[2];
      int c = 0;
      for (int p = lane; p < nt; p += 32) {
        long long v;
        if (grid_cell(a.g, (float)(sx[p] + tx), (float)(sy[p] + ty), (float)(sz[p] + tz), &v)) c += (int)((__ldg(&a.g.bits[v >> 5]) >> (v & 31)) & 1u);
      }
      for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
      if (lane == 0) cnt[j] += c;   // (translation j belongs to this warp alone)
    }
  }
  __syncthreads();
  if (threadIdx.x < RELOC_GROUP && l0 + (int)threadIdx.x < a.n_lat) a.scores[(size_t)r * a.n_lat + l0 + threadIdx.x] = cnt[threadIdx.x];
}

// h is a peak iff score(h) >= 1 and h comes first in (score descending, index ascending) among its lattice Chebyshev-1 neighbours (clipped at the
// border) at rotations r - 1, r, r + 1 (wrapped when cyclic and n_rot >= 3).  Peaks are appended as keys score << 32 | (2^32 - 1 - h).
__global__ void reloc_peak_kernel(const int32_t* __restrict__ scores, int nt0, int nt1, int nt2, int n_rot, int cyclic, int H, unsigned long long* __restrict__ peaks,
                                  int* __restrict__ count) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= H) return;
  const int s = scores[h];
  if (s < 1) return;
  const int n_lat = nt0 * nt1 * nt2;
  const int r = h / n_lat, l = h - r * n_lat, i = l % nt0, j = (l / nt0) % nt1, k = l / (nt0 * nt1);
  const bool wrap = cyclic && n_rot >= 3;
  for (int dr = -1; dr <= 1; dr++) {
    int rr = r + dr;
    if (wrap) rr = (rr + n_rot) % n_rot;
    else if (rr < 0 || rr >= n_rot) continue;
    for (int dk = -1; dk <= 1; dk++) {
      const int kk = k + dk; if (kk < 0 || kk >= nt2) continue;
      for (int dj = -1; dj <= 1; dj++) {
        const int jj = j + dj; if (jj < 0 || jj >= nt1) continue;
        for (int di = -1; di <= 1; di++) {
          const int ii = i + di; if (ii < 0 || ii >= nt0) continue;
          const int h2 = ii + nt0 * (jj + nt1 * kk) + n_lat * rr;
          if (h2 == h) continue;
          const int s2 = scores[h2];
          if (s2 > s || (s2 == s && h2 < h)) return;
        }
      }
    }
  }
  peaks[atomicAdd(count, 1)] = ((unsigned long long)(unsigned)s << 32) | (unsigned long long)(0xffffffffu - (unsigned)h);
}

// The first K peaks in (score descending, index ascending) order, i.e. the K largest keys: K rounds of a block-wide maximum below the last one.
__global__ void __launch_bounds__(1024) reloc_select_kernel(const unsigned long long* __restrict__ peaks, int* __restrict__ counts, int K, unsigned long long* __restrict__ cand) {
  __shared__ unsigned long long red[32];
  const int n = counts[0];
  unsigned long long bound = ~0ull;
  int k = 0;
  for (; k < K; k++) {
    unsigned long long best = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) { const unsigned long long v = peaks[i]; if (v < bound && v > best) best = v; }
    for (int o = 16; o > 0; o >>= 1) { const unsigned long long w = __shfl_xor_sync(0xffffffffu, best, o); best = w > best ? w : best; }
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = best;
    __syncthreads();
    best = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) best = red[w] > best ? red[w] : best;
    if (best == 0) break;   // (keys of peaks are > 0: score >= 1)
    if (threadIdx.x == 0) cand[k] = best;
    bound = best;
  }
  if (threadIdx.x == 0) counts[1] = k;
}

__global__ void reloc_gather_kernel(const float4* __restrict__ src, const int* __restrict__ idx, int n, float4* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[idx[i]];
}

void index_layout(ll_reloc_index* x, Carve& c) {
  x->bits = c.take<uint32_t>((size_t)x->n_words); x->scores = c.take<int32_t>(x->max_hyp); x->peaks = c.take<unsigned long long>(x->max_hyp);
  x->counts = c.take<int>(2); x->cand = c.take<unsigned long long>(LL_MAX_BATCH); x->pts = c.take<float4>(LL_RELOC_MAX_SCORE_POINTS);
  x->rot = c.take<double>((size_t)x->max_hyp * 4);
}

int check_map(ll_ctx* ctx, const ll_map* map) {
  if (map->world > 1) { ctx->set_error("relocalization needs the whole map: a sharded map is refused"); return LL_ERR_INVALID; }
  return LL_OK;
}

// A build's checks, then the map's grid into b (only on success): lo = the minimum of the finite bounding box both trees keep (d_bbox), dims_a =
// floor((hi_a - lo_a) / res) + 1 + 2 pad.  A map without a finite point: LL_ERR_INVALID; more than 2^30 voxels: LL_ERR_CAPACITY.
int build_grid(ll_ctx* ctx, const ll_map* map, float res, int pad, bool pad_ok, const char* pad_error, int max_hypotheses, RelocBase* b) {
  LL_TRY(check_map(ctx, map));
  if (!(res > 0.f) || !std::isfinite(res)) { ctx->set_error("res must be a finite value > 0"); return LL_ERR_INVALID; }
  if (!pad_ok) { ctx->set_error(pad_error); return LL_ERR_INVALID; }
  if (max_hypotheses < 1 || max_hypotheses > RELOC_MAX_HYP) { ctx->set_error("max_hypotheses must be 1 ... 2^24"); return LL_ERR_INVALID; }
  cudaSetDevice(ctx->device);
  cudaStream_t s = ctx->stream;
  float bb[2][6];
  for (int c = 0; c < 2; c++) if (map->tree[c].n_src > 0) LL_CUDA(ctx, cudaMemcpyAsync(bb[c], map->tree[c].d_bbox, sizeof(bb[c]), cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  bool any = false;
  for (int c = 0; c < 2; c++) {
    if (map->tree[c].n_src <= 0) continue;
    bool ok = true;
    for (int a = 0; a < 3; a++) ok = ok && std::isfinite(bb[c][a]) && std::isfinite(bb[c][3 + a]) && bb[c][a] <= bb[c][3 + a];
    if (!ok) continue;   // no finite point in this cloud
    any = true;
    for (int a = 0; a < 3; a++) { lo[a] = std::min(lo[a], bb[c][a]); hi[a] = std::max(hi[a], bb[c][3 + a]); }
  }
  if (!any) { ctx->set_error("the map has no finite point"); return LL_ERR_INVALID; }
  int dims[3];
  double nv = 1.0;
  for (int a = 0; a < 3; a++) {
    const double d = std::floor(((double)hi[a] - (double)lo[a]) / (double)res) + 1.0 + 2.0 * pad;
    if (!(d <= (double)RELOC_MAX_VOXELS)) { ctx->set_error("more than 2^30 voxels"); return LL_ERR_CAPACITY; }
    dims[a] = (int)d; nv *= d;
  }
  if (nv > (double)RELOC_MAX_VOXELS) { ctx->set_error("more than 2^30 voxels"); return LL_ERR_CAPACITY; }
  b->device = ctx->device; b->max_hyp = max_hypotheses; b->n_vox = (long long)dims[0] * dims[1] * dims[2];
  b->grid = {nullptr, {dims[0], dims[1], dims[2]}, {(double)lo[0], (double)lo[1], (double)lo[2]}, (double)res, pad};
  return LL_OK;
}

int check_device(ll_ctx* ctx, const RelocBase* b, const char* noun) {
  if (b->device != ctx->device) { ctx->set_error(std::string(noun) + " and context are on different devices"); return LL_ERR_INVALID; }
  return LL_OK;
}

// A relocalization's first checks: the map is whole, b (the "index" / "field") was built on it as it is now, and b is on the context's device.
int check_built_on(ll_ctx* ctx, const RelocBase* b, const ll_map* map, const char* noun) {
  LL_TRY(check_map(ctx, map));
  if (b->map != map || b->src[0] != map->tree[0].src || b->src[1] != map->tree[1].src || b->n_src[0] != map->tree[0].n_src || b->n_src[1] != map->tree[1].n_src) {
    ctx->set_error(std::string("the ") + noun + " was built on another map (or the map was rebuilt since)"); return LL_ERR_INVALID;
  }
  return check_device(ctx, b, noun);
}

bool unit_quaternions(ll_ctx* ctx, const double* rot, int n, const char* what) {
  for (int r = 0; r < n; r++) {
    const double* q = rot + 4 * r;
    const double n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
    if (!(std::fabs(std::sqrt(n2) - 1.0) <= 1e-6)) { ctx->set_error(std::string(what) + " " + std::to_string(r) + " is not a unit quaternion"); return false; }
  }
  return true;
}

// The configuration's hypothesis count (*H) after every check of ll_reloc_cfg except max_candidates.
int check_cfg(ll_ctx* ctx, int max_hyp, const ll_reloc_cfg* cfg, long long* H) {
  if (!cfg->rot_wxyz) { ctx->set_error("null rotation array"); return LL_ERR_INVALID; }
  if (cfg->n_rot < 1 || cfg->nt[0] < 1 || cfg->nt[1] < 1 || cfg->nt[2] < 1) { ctx->set_error("n_rot and nt must be >= 1"); return LL_ERR_INVALID; }
  for (int a = 0; a < 3; a++)
    if (!std::isfinite(cfg->t0[a]) || !std::isfinite(cfg->step[a])) { ctx->set_error("non-finite lattice origin or step"); return LL_ERR_INVALID; }
  const long long h = (long long)cfg->n_rot * cfg->nt[0] * cfg->nt[1] * cfg->nt[2];
  if ((long long)cfg->nt[0] * cfg->nt[1] * cfg->nt[2] > max_hyp || h > max_hyp) {
    ctx->set_error("more hypotheses than the index's max_hypotheses (" + std::to_string(max_hyp) + ")"); return LL_ERR_INVALID;
  }
  if (!unit_quaternions(ctx, cfg->rot_wxyz, cfg->n_rot, "rotation")) return LL_ERR_INVALID;
  *H = h;
  return LL_OK;
}

int check_points(ll_ctx* ctx, const void* pts, size_t n, int fmt, int where, const char* what) {
  if (fmt != LL_FMT_XYZI16 && fmt != LL_FMT_PCL32 && fmt != LL_FMT_STRIDED) { ctx->set_error("unknown point format"); return LL_ERR_INVALID; }
  if (where != LL_HOST && where != LL_DEVICE) { ctx->set_error("unknown memory kind"); return LL_ERR_INVALID; }
  if (!pts && n) { ctx->set_error(std::string("null ") + what); return LL_ERR_INVALID; }
  return LL_OK;
}

// The last checks of both relocalizations: the template's gate, the score points' count and the batch's capacity for K items of M features.
int check_refinement(ll_ctx* ctx, const ll_reg_state* tmpl, size_t n_score, const char* score_what, int K, size_t M) {
  if (tmpl->current_frame_index <= tmpl->mapping_init_accumulate_frames) {
    ctx->set_error("the template's frame index is at or below mapping_init_accumulate_frames: every refinement would skip the ICP (:199)"); return LL_ERR_INVALID;
  }
  if (n_score > LL_RELOC_MAX_SCORE_POINTS) { ctx->set_error(std::string("more than LL_RELOC_MAX_SCORE_POINTS ") + score_what); return LL_ERR_CAPACITY; }
  if ((size_t)K * M > (size_t)ctx->cfg.max_features) { ctx->set_error("K x the features (" + std::to_string((size_t)K * M) + ") exceed max_features"); return LL_ERR_CAPACITY; }
  int Ms[LL_MAX_BATCH]; for (int j = 0; j < K; j++) Ms[j] = (int)M;
  return solve_capacity(ctx, K, Ms, tmpl->if_motion_deblur ? 1 : 0);
}

// Hypothesis h = i + nt0 (j + nt1 k) + n_lat r of a lattice: q = rotation r of rot, t = t0 + (i, j, k) step.
void lattice_pose(const double* rot, const double* t0, const double* step, const int* nt, int h, double* q, double* t) {
  const int n_lat = nt[0] * nt[1] * nt[2];
  const int r = h / n_lat, l = h - r * n_lat, li[3] = {l % nt[0], (l / nt[0]) % nt[1], l / (nt[0] * nt[1])};
  for (int k = 0; k < 4; k++) q[k] = rot[4 * r + k];
  for (int k = 0; k < 3; k++) t[k] = t0[k] + (double)li[k] * step[k];
}

// The peaks of the H scores in b->scores, then the first K of them (*n) into cand: score, hypothesis and its pose (lattice_pose of cfg).
template <typename Cand> int coarse_candidates(ll_ctx* ctx, RelocBase* b, const ll_reloc_cfg* cfg, long long H, int K, Cand* cand, int* n) {
  cudaStream_t s = ctx->stream;
  LL_CUDA(ctx, cudaMemsetAsync(b->counts, 0, 2 * sizeof(int), s));
  reloc_peak_kernel<<<(unsigned)((H + 255) / 256), 256, 0, s>>>(b->scores, cfg->nt[0], cfg->nt[1], cfg->nt[2], cfg->n_rot, cfg->rot_cyclic ? 1 : 0, (int)H, b->peaks, b->counts);
  reloc_select_kernel<<<1, 1024, 0, s>>>(b->peaks, b->counts, K, b->cand);
  ctx->launches += 2;
  LL_CUDA(ctx, cudaGetLastError());
  unsigned long long keys[LL_MAX_BATCH]; int cnt[2] = {0, 0};
  LL_CUDA(ctx, cudaMemcpyAsync(cnt, b->counts, sizeof(cnt), cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaMemcpyAsync(keys, b->cand, sizeof(keys), cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  *n = cnt[1];
  for (int j = 0; j < *n; j++) {
    cand[j].score = (int32_t)(keys[j] >> 32); cand[j].hypothesis = (int)(0xffffffffu - (unsigned)(keys[j] & 0xffffffffu));
    lattice_pose(cfg->rot_wxyz, cfg->t0, cfg->step, cfg->nt, cand[j].hypothesis, cand[j].q_wxyz, cand[j].t);
  }
  return LL_OK;
}

// One registration batch of the same features, item j the template at seed pose (q[j], t[j]) with the identity increment.
int refine(ll_ctx* ctx, const ll_map* map, int n, const double* const* q, const double* const* t, const ll_reg_state* tmpl, const void* corner,
           size_t n_corner, const void* surf, size_t n_surf, int fmt, int where, ll_reg_result* refined, int* item_status) {
  ll_reg_state in[LL_MAX_BATCH];
  const void* cs[LL_MAX_BATCH]; const void* ss[LL_MAX_BATCH]; size_t ncs[LL_MAX_BATCH], nss[LL_MAX_BATCH];
  for (int j = 0; j < n; j++) {
    in[j] = *tmpl;
    for (int k = 0; k < 4; k++) { in[j].q_w_last[k] = q[j][k]; in[j].q_w_curr[k] = q[j][k]; }
    for (int k = 0; k < 3; k++) { in[j].t_w_last[k] = t[j][k]; in[j].t_w_curr[k] = t[j][k]; }
    for (int k = 0; k < 7; k++) in[j].para_buffer_incremental[k] = k == 3 ? 1.0 : 0.0;
    cs[j] = corner; ss[j] = surf; ncs[j] = n_corner; nss[j] = n_surf;
  }
  return ll_register_batch(ctx, map, n, cs, ncs, ss, nss, fmt, where, in, refined, item_status);
}

// Upload of the score points and the rotations, then the score kernel: scores[0 .. H) of the index, on the context's stream.
int enqueue_scores(ll_ctx* ctx, ll_reloc_index* idx, const void* pts, size_t n, int fmt, int where, const ll_reloc_cfg* cfg) {
  cudaStream_t s = ctx->stream;
  LL_TRY(upload_cloud(ctx, s, pts, n, fmt, where, idx->pts));
  LL_CUDA(ctx, cudaMemcpyAsync(idx->rot, cfg->rot_wxyz, (size_t)cfg->n_rot * 4 * sizeof(double), cudaMemcpyHostToDevice, s));
  ScoreArgs a;
  a.g = idx->grid; a.pts = idx->pts; a.n_pts = (int)n; a.rot = idx->rot; a.scores = idx->scores;
  for (int k = 0; k < 3; k++) { a.t0[k] = cfg->t0[k]; a.step[k] = cfg->step[k]; a.nt[k] = cfg->nt[k]; }
  a.n_lat = cfg->nt[0] * cfg->nt[1] * cfg->nt[2];
  a.blocks_per_rot = ll_div_up(a.n_lat, RELOC_GROUP);
  const long long blocks = (long long)cfg->n_rot * a.blocks_per_rot;
  reloc_score_kernel<<<(unsigned)blocks, 256, 0, s>>>(a); ctx->launches++;
  LL_CUDA(ctx, cudaGetLastError());
  return LL_OK;
}

// ------------------------------------------------------------------------------------------------ class-aware distance fields
__global__ void reloc_field_mark_kernel(const float4* __restrict__ src, int n, RelocGrid g, uint8_t* __restrict__ occ) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 p = src[i];
  if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) return;
  long long v;
  if (grid_cell(g, p.x, p.y, p.z, &v)) occ[v] = 1;
}

// One separable pass of the truncated squared distance transform along `axis`, one thread per voxel.  The first pass reads occupancy:
// min over |k| <= T of (occ(v + k e) ? k^2 : T^2); each later pass min over |k| <= T of in(v + k e) + k^2.  Voxels past the border are absent,
// every result is clamped to T^2.  A term with |k| > T is at least T^2 + 1, so the truncated window gives the exact transform.
__global__ void reloc_edt_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int d0, int d1, int d2, int axis, int T, int first, long long n_vox) {
  const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vox) return;
  const long long yz = v / d0;
  const int x = (int)(v - yz * d0), y = (int)(yz % d1), z = (int)(yz / d1);
  const int c = axis == 0 ? x : (axis == 1 ? y : z), D = axis == 0 ? d0 : (axis == 1 ? d1 : d2);
  const long long stride = axis == 0 ? 1 : (axis == 1 ? (long long)d0 : (long long)d0 * d1);
  const int T2 = T * T;
  int best = T2;
  for (int k = max(c - T, 0) - c; k <= min(c + T, D - 1) - c; k++) {
    const int g = (int)in[v + (long long)k * stride];
    best = min(best, first ? (g ? k * k : T2) : g + k * k);
  }
  out[v] = (uint8_t)best;
}

struct FieldScoreArgs {
  RelocGrid g; const uint8_t* d2[2]; const float4* pts[2]; int n_pts[2];
  const double* rot;   // [n_groups x n_rot x 4]
  const double* t0;    // [n_groups x 3]
  double step[3]; int nt[3]; int n_rot, n_lat, blocks_per_rot;
  int32_t* scores;     // [n_groups x n_rot x n_lat]
};
// The layout of reloc_score_kernel with groups: CTA = one rotation of one group x RELOC_GROUP consecutive lattice points of that group's lattice.
// A score point of class c adds T^2 - D_c(cell) where its p_w lands inside the grid.  Global rotation gr = r + n_rot * group; the score of
// hypothesis l + n_lat * r of the group is at scores[gr * n_lat + l].
__global__ void __launch_bounds__(256) reloc_field_score_kernel(FieldScoreArgs a) {
  __shared__ double sx[RELOC_TILE], sy[RELOC_TILE], sz[RELOC_TILE];
  __shared__ int acc[RELOC_GROUP];
  const int gr = blockIdx.x / a.blocks_per_rot, l0 = (blockIdx.x - gr * a.blocks_per_rot) * RELOC_GROUP, grp = gr / a.n_rot;
  const double q[4] = {a.rot[4 * gr], a.rot[4 * gr + 1], a.rot[4 * gr + 2], a.rot[4 * gr + 3]};
  const double o[3] = {a.t0[3 * grp], a.t0[3 * grp + 1], a.t0[3 * grp + 2]};
  const int T2 = a.g.dilate * a.g.dilate;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, n_warps = blockDim.x >> 5;
  if (threadIdx.x < RELOC_GROUP) acc[threadIdx.x] = 0;
  for (int cls = 0; cls < 2; cls++) {
    const uint8_t* __restrict__ f = a.d2[cls];
    const float4* __restrict__ pts = a.pts[cls];
    for (int base = 0; base < a.n_pts[cls]; base += RELOC_TILE) {
      const int nt = min(RELOC_TILE, a.n_pts[cls] - base);
      __syncthreads();
      for (int i = threadIdx.x; i < nt; i += blockDim.x) {
        const float4 p = pts[base + i];
        double ox = CUDART_NAN, oy = CUDART_NAN, oz = CUDART_NAN;   // a point with a non-finite coordinate never scores
        if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) qrot_d(q, (double)p.x, (double)p.y, (double)p.z, ox, oy, oz);
        sx[i] = ox; sy[i] = oy; sz[i] = oz;
      }
      __syncthreads();
      for (int j = warp; j < RELOC_GROUP; j += n_warps) {
        const int l = l0 + j;
        if (l >= a.n_lat) break;
        const int i0 = l % a.nt[0], i1 = (l / a.nt[0]) % a.nt[1], i2 = l / (a.nt[0] * a.nt[1]);
        const double tx = o[0] + (double)i0 * a.step[0], ty = o[1] + (double)i1 * a.step[1], tz = o[2] + (double)i2 * a.step[2];
        int s = 0;
        for (int p = lane; p < nt; p += 32) {
          long long v;
          if (grid_cell(a.g, (float)(sx[p] + tx), (float)(sy[p] + ty), (float)(sz[p] + tz), &v)) s += T2 - (int)__ldg(&f[v]);
        }
        for (int k = 16; k > 0; k >>= 1) s += __shfl_xor_sync(0xffffffffu, s, k);
        if (lane == 0) acc[j] += s;   // (translation j belongs to this warp alone)
      }
    }
  }
  __syncthreads();
  if (threadIdx.x < RELOC_GROUP && l0 + (int)threadIdx.x < a.n_lat) a.scores[(size_t)gr * a.n_lat + l0 + threadIdx.x] = acc[threadIdx.x];
}

// Each group's pick: its first hypothesis in (score descending, index ascending), as the key score << 32 | (2^32 - 1 - index).  One CTA per group
// of `per_group` scores (all >= 0, so every key is > 0).
__global__ void __launch_bounds__(1024) reloc_pick_kernel(const int32_t* __restrict__ scores, int per_group, unsigned long long* __restrict__ picks) {
  __shared__ unsigned long long red[32];
  const int32_t* s = scores + (size_t)blockIdx.x * per_group;
  unsigned long long best = 0;
  for (int i = threadIdx.x; i < per_group; i += blockDim.x) {
    const unsigned long long k = ((unsigned long long)(unsigned)s[i] << 32) | (unsigned long long)(0xffffffffu - (unsigned)i);
    best = k > best ? k : best;
  }
  for (int o = 16; o > 0; o >>= 1) { const unsigned long long w = __shfl_xor_sync(0xffffffffu, best, o); best = w > best ? w : best; }
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) best = red[w] > best ? red[w] : best;
    picks[blockIdx.x] = best;
  }
}

void field_layout(ll_reloc_field* f, Carve& c) {
  for (int k = 0; k < 2; k++) f->d2[k] = c.take<uint8_t>((size_t)f->n_vox);
  f->scores = c.take<int32_t>(f->max_hyp); f->peaks = c.take<unsigned long long>(f->max_hyp); f->counts = c.take<int>(2);
  f->cand = c.take<unsigned long long>(LL_MAX_BATCH); f->fine = c.take<int32_t>(f->max_hyp); f->picks = c.take<unsigned long long>(LL_MAX_BATCH);
  f->verify = c.take<int32_t>(LL_MAX_BATCH);
  for (int k = 0; k < 2; k++) f->pts[k] = c.take<float4>(LL_RELOC_MAX_SCORE_POINTS);
  f->rot = c.take<double>((size_t)f->max_hyp * 4); f->t0 = c.take<double>(LL_MAX_BATCH * 3);
}

// The rotations (n_groups x n_rot, host) and origins (n_groups, host) of the groups uploaded, then the score kernel: out[0 .. n_groups x n_rot x
// n_lat) on the context's stream.  The score points are already on the device.
int enqueue_field_scores(ll_ctx* ctx, ll_reloc_field* f, int n_sc, int n_ss, int n_groups, const double* rot, int n_rot, const double* t0,
                         const double step[3], const int nt[3], int32_t* out) {
  cudaStream_t s = ctx->stream;
  LL_CUDA(ctx, cudaMemcpyAsync(f->rot, rot, (size_t)n_groups * n_rot * 4 * sizeof(double), cudaMemcpyHostToDevice, s));
  LL_CUDA(ctx, cudaMemcpyAsync(f->t0, t0, (size_t)n_groups * 3 * sizeof(double), cudaMemcpyHostToDevice, s));
  FieldScoreArgs a;
  a.g = f->grid;
  for (int c = 0; c < 2; c++) { a.d2[c] = f->d2[c]; a.pts[c] = f->pts[c]; }
  a.n_pts[0] = n_sc; a.n_pts[1] = n_ss; a.rot = f->rot; a.t0 = f->t0; a.scores = out;
  for (int k = 0; k < 3; k++) { a.step[k] = step[k]; a.nt[k] = nt[k]; }
  a.n_rot = n_rot; a.n_lat = nt[0] * nt[1] * nt[2];
  a.blocks_per_rot = ll_div_up(a.n_lat, RELOC_GROUP);
  const long long blocks = (long long)n_groups * n_rot * a.blocks_per_rot;
  reloc_field_score_kernel<<<(unsigned)blocks, 256, 0, s>>>(a); ctx->launches++;
  LL_CUDA(ctx, cudaGetLastError());
  return LL_OK;
}

template <typename T> void release(T* x) { if (!x) return; cudaSetDevice(x->device); x->storage.release(); delete x; }

}  // namespace

void quat_mul(const double* a, const double* b, double* o) {
  o[0] = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  o[1] = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  o[2] = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
  o[3] = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
}

// The live points of a cell map in store order (cm_live_points, cellmap.cu) are gathered here.
int launch_gather_points(ll_ctx* ctx, cudaStream_t s, const float4* src, const int* idx, int n, float4* dst) {
  if (n <= 0) return LL_OK;
  reloc_gather_kernel<<<ll_div_up(n, 256), 256, 0, s>>>(src, idx, n, dst); ctx->launches++;
  LL_CUDA(ctx, cudaGetLastError());
  return LL_OK;
}

ll_reloc_field* reloc_field_create(int device) { ll_reloc_field* f = new ll_reloc_field(); f->device = device; return f; }
size_t reloc_field_storage_cap(const ll_reloc_field* f) { return f->storage.cap; }

// The storage of a field of n_vox voxels and max_hyp hypotheses, and the context's scratch for its build: allocated now, so that a build into f
// within these sizes allocates nothing.
int reloc_field_reserve(ll_ctx* ctx, ll_reloc_field* f, long long n_vox, int max_hyp) {
  ll_reloc_field x; x.n_vox = n_vox; x.max_hyp = max_hyp;
  LL_CUDA(ctx, f->storage.reserve_floor(layout_bytes([&](Carve& c) { field_layout(&x, c); })));
  LL_CUDA(ctx, ctx->scratch.reserve_floor((size_t)n_vox));
  return LL_OK;
}

// ll_reloc_field_build into an existing field, reusing its storage when it is large enough (ll_reloc_field_build: a new one; the streaming
// mapper's recovery: its own, once per loss episode).  On an error f holds no field (its map is cleared).
int reloc_field_build_into(ll_ctx* ctx, const ll_map* map, float res, int trunc, int max_hypotheses, ll_reloc_field* f) {
  f->map = nullptr; f->src[0] = f->src[1] = nullptr; f->n_src[0] = f->n_src[1] = 0;
  LL_TRY(build_grid(ctx, map, res, trunc, trunc >= 1 && trunc <= RELOC_MAX_TRUNC, "trunc must be 1 ... 15", max_hypotheses, f));
  cudaStream_t s = ctx->stream;
  { const cudaError_t e = f->storage.carve([&](Carve& c) { field_layout(f, c); });
    if (e != cudaSuccess) { ctx->set_error(std::string("field allocation: ") + cudaGetErrorString(e)); return LL_ERR_CUDA; } }
  uint8_t* tmp = nullptr;   // occupancy, then the pass between y and z
  { const cudaError_t e = ctx->scratch.carve([&](Carve& c) { tmp = c.take<uint8_t>((size_t)f->n_vox); });
    if (e != cudaSuccess) { ctx->set_error(std::string("field scratch: ") + cudaGetErrorString(e)); return LL_ERR_CUDA; } }
  int st = LL_OK;
  auto cu = [&](cudaError_t e) { if (e != cudaSuccess && st == LL_OK) { ctx->set_error(std::string("field build: ") + cudaGetErrorString(e)); st = LL_ERR_CUDA; } };
  const unsigned blocks = (unsigned)((f->n_vox + 255) / 256);
  for (int c = 0; c < 2; c++) {
    const BucketTree& t = map->tree[c];
    cu(cudaMemsetAsync(tmp, 0, (size_t)f->n_vox, s));
    if (t.n_src > 0) { reloc_field_mark_kernel<<<ll_div_up(t.n_src, 256), 256, 0, s>>>(t.src, t.n_src, f->grid, tmp); ctx->launches++; }
    uint8_t* io[3][2] = {{tmp, f->d2[c]}, {f->d2[c], tmp}, {tmp, f->d2[c]}};
    for (int a = 0; a < 3; a++) { reloc_edt_kernel<<<blocks, 256, 0, s>>>(io[a][0], io[a][1], f->grid.dims[0], f->grid.dims[1], f->grid.dims[2], a, trunc, a == 0 ? 1 : 0, f->n_vox); ctx->launches++; }
  }
  cu(cudaGetLastError());
  cu(cudaStreamSynchronize(s));
  if (st != LL_OK) return st;
  f->map = map;
  for (int c = 0; c < 2; c++) { f->src[c] = map->tree[c].src; f->n_src[c] = map->tree[c].n_src; }
  return LL_OK;
}

extern "C" {

int ll_reloc_index_build(ll_ctx* ctx, const ll_map* map, float res, int dilate, int max_hypotheses, ll_reloc_index** out) {
  if (!ctx || !map || !out) return LL_ERR_INVALID;
  *out = nullptr;
  RelocBase base;
  LL_TRY(build_grid(ctx, map, res, dilate, dilate >= 0 && dilate <= RELOC_MAX_DILATE, "dilate must be 0 ... 4", max_hypotheses, &base));
  cudaStream_t s = ctx->stream;
  ll_reloc_index* x = new ll_reloc_index{base};
  x->map = map;
  for (int c = 0; c < 2; c++) { x->src[c] = map->tree[c].src; x->n_src[c] = map->tree[c].n_src; }
  x->n_words = (x->n_vox + 31) / 32;
  auto fail = [&](int st) { x->storage.release(); delete x; return st; };
  { const cudaError_t e = x->storage.carve([&](Carve& c) { index_layout(x, c); });
    if (e != cudaSuccess) { ctx->set_error(std::string("index allocation: ") + cudaGetErrorString(e)); return fail(LL_ERR_CUDA); } }
  // occupancy into `occ` (the index itself when nothing is dilated), then x, y, z passes ping-ponging with the context's scratch
  uint32_t* tmp = nullptr;
  if (dilate > 0) {
    const cudaError_t e = ctx->scratch.carve([&](Carve& c) { tmp = c.take<uint32_t>((size_t)x->n_words); });
    if (e != cudaSuccess) { ctx->set_error(std::string("index scratch: ") + cudaGetErrorString(e)); return fail(LL_ERR_CUDA); }
  }
  uint32_t* occ = dilate > 0 ? tmp : x->bits;
  x->grid.bits = x->bits;
  int st = LL_OK;
  auto cu = [&](cudaError_t e) { if (e != cudaSuccess && st == LL_OK) { ctx->set_error(std::string("index build: ") + cudaGetErrorString(e)); st = LL_ERR_CUDA; } };
  cu(cudaMemsetAsync(occ, 0, (size_t)x->n_words * 4, s));
  for (const BucketTree& t : map->tree) if (t.n_src > 0) { reloc_mark_kernel<<<ll_div_up(t.n_src, 256), 256, 0, s>>>(t.src, t.n_src, base.grid, occ); ctx->launches++; }
  if (dilate > 0) {
    const long long threads = x->n_words * 32;
    const unsigned blocks = (unsigned)((threads + 255) / 256);
    uint32_t* io[3][2] = {{tmp, x->bits}, {x->bits, tmp}, {tmp, x->bits}};
    for (int a = 0; a < 3; a++) { reloc_dilate_kernel<<<blocks, 256, 0, s>>>(io[a][0], io[a][1], x->grid.dims[0], x->grid.dims[1], x->grid.dims[2], a, dilate, x->n_vox, x->n_words); ctx->launches++; }
  }
  cu(cudaGetLastError());
  cu(cudaStreamSynchronize(s));
  if (st != LL_OK) return fail(st);
  *out = x;
  return LL_OK;
}

void ll_reloc_index_release(ll_reloc_index* idx) { release(idx); }

int ll_reloc_index_read(const ll_reloc_index* idx, int dims[3], float lo[3], uint32_t* words, size_t cap_words) {
  if (!idx) return LL_ERR_INVALID;
  if (dims) for (int a = 0; a < 3; a++) dims[a] = idx->grid.dims[a];
  if (lo) for (int a = 0; a < 3; a++) lo[a] = (float)idx->grid.lo[a];
  if (!words) return LL_OK;
  if (cap_words < (size_t)idx->n_words) return LL_ERR_CAPACITY;
  cudaSetDevice(idx->device);
  if (cudaMemcpy(words, idx->bits, (size_t)idx->n_words * 4, cudaMemcpyDeviceToHost) != cudaSuccess) return LL_ERR_CUDA;
  return LL_OK;
}

int ll_reloc_scores(ll_ctx* ctx, const ll_reloc_index* cidx, const void* score_pts, size_t n_score, int fmt, int where, const ll_reloc_cfg* cfg, int32_t* scores) {
  if (!ctx || !cidx || !cfg || !scores) return LL_ERR_INVALID;
  ll_reloc_index* idx = const_cast<ll_reloc_index*>(cidx);   // (its work buffers; the index itself is not changed)
  LL_TRY(check_points(ctx, score_pts, n_score, fmt, where, "score points"));
  long long H = 0;
  LL_TRY(check_cfg(ctx, idx->max_hyp, cfg, &H));
  if (n_score > LL_RELOC_MAX_SCORE_POINTS) { ctx->set_error("more than LL_RELOC_MAX_SCORE_POINTS score points"); return LL_ERR_CAPACITY; }
  LL_TRY(check_device(ctx, idx, "index"));
  cudaSetDevice(ctx->device);
  LL_TRY(enqueue_scores(ctx, idx, score_pts, n_score, fmt, where, cfg));
  LL_CUDA(ctx, cudaMemcpyAsync(scores, idx->scores, (size_t)H * 4, cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return LL_OK;
}

int ll_relocalize(ll_ctx* ctx, const ll_map* map, const ll_reloc_index* cidx, const void* score_pts, size_t n_score, const void* corner, size_t n_corner,
                  const void* surf, size_t n_surf, int fmt, int where, const ll_reloc_cfg* cfg, const ll_reg_state* tmpl, ll_reloc_candidate* cand,
                  ll_reg_result* refined, int* item_status, int* n_cand, int* best) {
  if (!ctx || !map || !cidx || !cfg || !tmpl || !cand || !refined || !item_status || !n_cand || !best) return LL_ERR_INVALID;
  ll_reloc_index* idx = const_cast<ll_reloc_index*>(cidx);
  *n_cand = 0; *best = -1;
  LL_TRY(check_built_on(ctx, idx, map, "index"));
  LL_TRY(check_points(ctx, score_pts, n_score, fmt, where, "score points"));
  LL_TRY(check_points(ctx, corner, n_corner, fmt, where, "corner features"));
  LL_TRY(check_points(ctx, surf, n_surf, fmt, where, "surface features"));
  long long H = 0;
  LL_TRY(check_cfg(ctx, idx->max_hyp, cfg, &H));
  const int K = cfg->max_candidates;
  if (K < 1 || K > LL_MAX_BATCH) { ctx->set_error("max_candidates must be 1 ... LL_MAX_BATCH"); return LL_ERR_INVALID; }
  LL_TRY(check_refinement(ctx, tmpl, n_score, "score points", K, n_corner + n_surf));
  cudaSetDevice(ctx->device);
  // scores -> peaks -> the first K peaks
  LL_TRY(enqueue_scores(ctx, idx, score_pts, n_score, fmt, where, cfg));
  int n = 0;
  LL_TRY(coarse_candidates(ctx, idx, cfg, H, K, cand, &n));
  if (n == 0) return LL_OK;
  // refinement: the candidates as the items of one registration batch, each seeded at its hypothesis
  const double* q[LL_MAX_BATCH]; const double* t[LL_MAX_BATCH];
  for (int j = 0; j < n; j++) { q[j] = cand[j].q_wxyz; t[j] = cand[j].t; }
  *n_cand = n;
  LL_TRY(refine(ctx, map, n, q, t, tmpl, corner, n_corner, surf, n_surf, fmt, where, refined, item_status));
  // the choice: the smallest inlier_threshold (:559) among the accepted registrations, ties to the lower rank
  for (int j = 0; j < n; j++) {
    const ll_reg_result& r = refined[j];
    if (item_status[j] != LL_OK || r.registered != 1 || r.status != 1) continue;
    if (*best < 0 || r.inlier_threshold < refined[*best].inlier_threshold) *best = j;
  }
  return LL_OK;
}

int ll_reloc_field_build(ll_ctx* ctx, const ll_map* map, float res, int trunc, int max_hypotheses, ll_reloc_field** out) {
  if (!ctx || !map || !out) return LL_ERR_INVALID;
  *out = nullptr;
  ll_reloc_field* f = reloc_field_create(ctx->device);
  const int st = reloc_field_build_into(ctx, map, res, trunc, max_hypotheses, f);
  if (st != LL_OK) { ll_reloc_field_release(f); return st; }
  *out = f;
  return LL_OK;
}

void ll_reloc_field_release(ll_reloc_field* field) { release(field); }

int ll_reloc_field_read(const ll_reloc_field* field, int which, int dims[3], float lo[3], uint8_t* d2, size_t cap) {
  if (!field || (which != 0 && which != 1)) return LL_ERR_INVALID;
  if (dims) for (int a = 0; a < 3; a++) dims[a] = field->grid.dims[a];
  if (lo) for (int a = 0; a < 3; a++) lo[a] = (float)field->grid.lo[a];
  if (!d2) return LL_OK;
  if (cap < (size_t)field->n_vox) return LL_ERR_CAPACITY;
  cudaSetDevice(field->device);
  if (cudaMemcpy(d2, field->d2[which], (size_t)field->n_vox, cudaMemcpyDeviceToHost) != cudaSuccess) return LL_ERR_CUDA;
  return LL_OK;
}

int ll_reloc_field_scores(ll_ctx* ctx, const ll_reloc_field* cfield, const void* score_corner, size_t n_sc, const void* score_surf, size_t n_ss, int fmt,
                          int where, const ll_reloc_cfg* cfg, int32_t* scores) {
  if (!ctx || !cfield || !cfg || !scores) return LL_ERR_INVALID;
  ll_reloc_field* f = const_cast<ll_reloc_field*>(cfield);   // (its work buffers; the fields themselves are not changed)
  LL_TRY(check_device(ctx, f, "field"));
  LL_TRY(check_points(ctx, score_corner, n_sc, fmt, where, "corner score points"));
  LL_TRY(check_points(ctx, score_surf, n_ss, fmt, where, "surface score points"));
  long long H = 0;
  LL_TRY(check_cfg(ctx, f->max_hyp, cfg, &H));
  if (std::max(n_sc, n_ss) > LL_RELOC_MAX_SCORE_POINTS) { ctx->set_error("more than LL_RELOC_MAX_SCORE_POINTS score points in a class"); return LL_ERR_CAPACITY; }
  cudaSetDevice(ctx->device);
  LL_TRY(upload_cloud(ctx, ctx->stream, score_corner, n_sc, fmt, where, f->pts[0]));
  LL_TRY(upload_cloud(ctx, ctx->stream, score_surf, n_ss, fmt, where, f->pts[1]));
  LL_TRY(enqueue_field_scores(ctx, f, (int)n_sc, (int)n_ss, 1, cfg->rot_wxyz, cfg->n_rot, cfg->t0, cfg->step, cfg->nt, f->scores));
  LL_CUDA(ctx, cudaMemcpyAsync(scores, f->scores, (size_t)H * 4, cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return LL_OK;
}

int ll_relocalize_field(ll_ctx* ctx, const ll_map* map, const ll_reloc_field* cfield, const void* score_corner, size_t n_sc, const void* score_surf,
                        size_t n_ss, const void* corner, size_t n_corner, const void* surf, size_t n_surf, int fmt, int where, const ll_reloc_cfg* coarse,
                        const ll_reloc_fine_cfg* fine, const ll_reg_state* tmpl, ll_reloc_field_candidate* cand, ll_reg_result* refined, int* item_status,
                        int* n_cand, int* best) {
  if (!ctx || !map || !cfield || !coarse || !fine || !tmpl || !cand || !refined || !item_status || !n_cand || !best) return LL_ERR_INVALID;
  ll_reloc_field* f = const_cast<ll_reloc_field*>(cfield);
  *n_cand = 0; *best = -1;
  LL_TRY(check_built_on(ctx, f, map, "field"));
  LL_TRY(check_points(ctx, score_corner, n_sc, fmt, where, "corner score points"));
  LL_TRY(check_points(ctx, score_surf, n_ss, fmt, where, "surface score points"));
  LL_TRY(check_points(ctx, corner, n_corner, fmt, where, "corner features"));
  LL_TRY(check_points(ctx, surf, n_surf, fmt, where, "surface features"));
  long long H = 0;
  LL_TRY(check_cfg(ctx, f->max_hyp, coarse, &H));
  const int K = coarse->max_candidates;
  if (K < 1 || K > LL_MAX_BATCH) { ctx->set_error("max_candidates must be 1 ... LL_MAX_BATCH"); return LL_ERR_INVALID; }
  // the fine search: K groups of n_rot x nt0 x nt1 x nt2 hypotheses, centred on each candidate
  if (!fine->rot_wxyz) { ctx->set_error("null fine rotation array"); return LL_ERR_INVALID; }
  if (fine->n_rot < 1 || fine->nt[0] < 1 || fine->nt[1] < 1 || fine->nt[2] < 1) { ctx->set_error("fine n_rot and nt must be >= 1"); return LL_ERR_INVALID; }
  for (int a = 0; a < 3; a++) {
    if (fine->nt[a] % 2 == 0) { ctx->set_error("fine nt must be odd (a lattice centred on the candidate)"); return LL_ERR_INVALID; }
    if (!std::isfinite(fine->step[a])) { ctx->set_error("non-finite fine step"); return LL_ERR_INVALID; }
  }
  const long long n_lat_f = (long long)fine->nt[0] * fine->nt[1] * fine->nt[2], H_f = n_lat_f * fine->n_rot;
  if (n_lat_f > f->max_hyp || H_f > f->max_hyp || (long long)K * H_f > f->max_hyp) {
    ctx->set_error("max_candidates x the fine hypotheses exceed the field's max_hypotheses (" + std::to_string(f->max_hyp) + ")"); return LL_ERR_INVALID;
  }
  if (!unit_quaternions(ctx, fine->rot_wxyz, fine->n_rot, "fine rotation")) return LL_ERR_INVALID;
  LL_TRY(check_refinement(ctx, tmpl, std::max(n_sc, n_ss), "score points in a class", K, n_corner + n_surf));
  cudaSetDevice(ctx->device);
  cudaStream_t s = ctx->stream;
  // 1. coarse: scores -> peaks -> the first K peaks
  LL_TRY(upload_cloud(ctx, ctx->stream, score_corner, n_sc, fmt, where, f->pts[0]));
  LL_TRY(upload_cloud(ctx, ctx->stream, score_surf, n_ss, fmt, where, f->pts[1]));
  LL_TRY(enqueue_field_scores(ctx, f, (int)n_sc, (int)n_ss, 1, coarse->rot_wxyz, coarse->n_rot, coarse->t0, coarse->step, coarse->nt, f->scores));
  int n = 0;
  LL_TRY(coarse_candidates(ctx, f, coarse, H, K, cand, &n));
  if (n == 0) return LL_OK;
  // 2. fine: group j = the rotations q_j (x) dq_r and the lattice origin t_j - ((nt - 1) / 2) step; its pick is its best hypothesis
  std::vector<double> rot_f((size_t)n * fine->n_rot * 4);
  double t0_f[LL_MAX_BATCH * 3];
  for (int j = 0; j < n; j++) {
    const ll_reloc_field_candidate& c = cand[j];
    for (int rr = 0; rr < fine->n_rot; rr++) quat_mul(c.q_wxyz, fine->rot_wxyz + 4 * rr, &rot_f[((size_t)j * fine->n_rot + rr) * 4]);
    for (int k = 0; k < 3; k++) t0_f[3 * j + k] = c.t[k] - (double)((fine->nt[k] - 1) / 2) * fine->step[k];
  }
  LL_TRY(enqueue_field_scores(ctx, f, (int)n_sc, (int)n_ss, n, rot_f.data(), fine->n_rot, t0_f, fine->step, fine->nt, f->fine));
  reloc_pick_kernel<<<n, 1024, 0, s>>>(f->fine, (int)H_f, f->picks); ctx->launches++;
  LL_CUDA(ctx, cudaGetLastError());
  unsigned long long picks[LL_MAX_BATCH];
  LL_CUDA(ctx, cudaMemcpyAsync(picks, f->picks, (size_t)n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  // 3. refinement: the picks as the items of one registration batch, seeded as ll_relocalize seeds its candidates
  const double* q[LL_MAX_BATCH]; const double* t[LL_MAX_BATCH];
  for (int j = 0; j < n; j++) {
    ll_reloc_field_candidate& c = cand[j];
    c.fine_score = (int32_t)(picks[j] >> 32); c.fine_index = (int)(0xffffffffu - (unsigned)(picks[j] & 0xffffffffu));
    lattice_pose(&rot_f[(size_t)j * fine->n_rot * 4], &t0_f[3 * j], fine->step, fine->nt, c.fine_index, c.fine_q_wxyz, c.fine_t);
    c.verify_score = 0; c.reserved = 0;
    q[j] = c.fine_q_wxyz; t[j] = c.fine_t;
  }
  *n_cand = n;
  LL_TRY(refine(ctx, map, n, q, t, tmpl, corner, n_corner, surf, n_surf, fmt, where, refined, item_status));
  // 4. verify: the same score at every refined pose (one group of one rotation and one translation each)
  double rot_v[LL_MAX_BATCH * 4], t0_v[LL_MAX_BATCH * 3];
  for (int j = 0; j < n; j++) {
    for (int k = 0; k < 4; k++) rot_v[4 * j + k] = refined[j].q_w_curr[k];
    for (int k = 0; k < 3; k++) t0_v[3 * j + k] = refined[j].t_w_curr[k];
  }
  const double step_v[3] = {0.0, 0.0, 0.0}; const int nt_v[3] = {1, 1, 1};
  LL_TRY(enqueue_field_scores(ctx, f, (int)n_sc, (int)n_ss, n, rot_v, 1, t0_v, step_v, nt_v, f->verify));
  int32_t ver[LL_MAX_BATCH];
  LL_CUDA(ctx, cudaMemcpyAsync(ver, f->verify, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  // the choice: the accepted item of the largest verify score, ties to the smaller inlier_threshold, then to the lower rank
  for (int j = 0; j < n; j++) {
    cand[j].verify_score = ver[j];
    const ll_reg_result& r = refined[j];
    if (item_status[j] != LL_OK || r.registered != 1 || r.status != 1) continue;
    if (*best < 0 || ver[j] > ver[*best] || (ver[j] == ver[*best] && r.inlier_threshold < refined[*best].inlier_threshold)) *best = j;
  }
  return LL_OK;
}

}  // extern "C"
