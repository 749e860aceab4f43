// Spinning-lidar front end on the device: the Velodyne branch of Laser_feature::laserCloudHandler (scan_line 16 / 64).
//
// Replaces, on the reference side (laser_feature_extractor.hpp):
//   removeNaNFromPointCloud + removeClosedPointCloud            :399-400, :211-240
//   ring, orientation unwrapping, relative time                  :403-504
//   ring-ordered concatenation, scanStartInd / scanEndInd         :510-521
//   curvature, occlusion and parallel-beam flags                  :524-598
//   per-ring 6 sub-scans: sort, sharp / flat picks, less flat     :631-768
//   per-ring VoxelGrid of the less-flat points                    :770-776
//
// Stages (one stream, no host synchronisation until the final count read-back):
//   filter (order-preserving compaction) -> ring + halfPassed (first-index reduction) -> stable bucketing by ring (radix sort of the ring id)
//   -> gather with relative time -> curvature, flags, gap cuts -> sub-scan sort (radix sort of sub-scan start << 32 | curvature bits, stable)
//   -> chains -> selection (one warp per chain) -> outputs -> less-flat compaction -> segmented VoxelGrid (one segment per ring).
// The selection is the only sequential part.  A pick marks its neighbours only up to the first consecutive squared gap > 0.05 (a "cut"), and
// sub-scans are visited in index order, so a pick affects only later sub-scans up to the next cut: consecutive sub-scans X, Y are independent
// when a cut lies in (ep_X, sp_Y].  The sub-scans split into chains at those cuts and each chain is one warp, visiting 32 candidates at a time.
//
// Deviations from the reference (DESIGN.md §4.7): the result is defined on the kept points only (the reference indexes the filtered cloud
// with the unfiltered size); the neighbour walks stop at the ends of the cloud; fewer than 5 kept points give empty feature clouds; points with
// a coordinate of magnitude above 1e36 are removed with the non-finite ones (no sum of the curvature can overflow, so it is never NaN).
// atan / atan2 are the correctly rounded float of the double functions, as everywhere else in this library.
// Compiled with -fmad=false: every float expression rounds like the scalar CPU code.
#include <cub/cub.cuh>
#include <cmath>
#include "common.cuh"
#include "kernels.cuh"

#define FULL 0xffffffffu
#define SPIN_PI 3.14159265358979323846
#define SPIN_MAX_COORD 1e36f
#define SPIN_SHARP_MAX 200
#define SPIN_FLAT_MAX 5
#define SPIN_SUB 6
#define SPIN_MAX_RINGS 64
#define SPIN_MAX_SUBS (SPIN_SUB * SPIN_MAX_RINGS)

// device meta block (one memset clears it)
struct SpinMeta {
  int nf;                        // filtered points
  int first_half;                // first filtered index whose first-branch orientation passes half a turn (INT_MAX: none)
  int ring_cnt[SPIN_MAX_RINGS];
  int ring_begin[SPIN_MAX_RINGS + 1];
  int sp[SPIN_MAX_SUBS], ep[SPIN_MAX_SUBS];
  int nsharp[SPIN_MAX_SUBS], nflat[SPIN_MAX_SUBS];
  int chain_first[SPIN_MAX_SUBS + 1];
  int lf_cnt[SPIN_MAX_RINGS], lf_end[SPIN_MAX_RINGS], vg_end[SPIN_MAX_RINGS];
  int nlf;                       // less-flat points before the VoxelGrid (DeviceSelect count)
  int counts[8];                 // N, sharp, less sharp, flat, less flat, chains, longest chain (points), less flat before the VoxelGrid
  int feat[4];                   // streaming mapper input: corners and surfaces after the mapping node's VoxelGrids, ll_f2ord of max_t, unused
};

struct ll_spin {
  ll_ctx* ctx = nullptr;
  ll_spin_cfg cfg = {};
  int rings = 16;
  int last_counts[8] = {0};
  int extracted = 0, last_n = 0;
  DevBuf arena, vg_scratch;
  int* pin = nullptr;            // pinned: SpinMeta::counts, then SpinMeta::feat (the streaming mapper's sweeps)
  // arena
  float4* in4; float4* filt; float4* cloud; int* rkey[2]; int* rval[2]; unsigned long long* ckey[2]; int* cval[2];
  float* curv; unsigned char* occl; unsigned char* beam; unsigned* picked; unsigned* picked0; unsigned* cut; signed char* label; short* sid;
  unsigned char* lfflag; int* sharp_idx; int* flat_idx;
  float4* out_sharp; float4* out_less_sharp; float4* out_flat; float4* lf_raw; float4* out_less_flat;
  SpinMeta* meta; char* tmp; size_t tmp_bytes = 0;
  // the streaming mapper's input (spin_sweep_enqueue): the mapping node's VoxelGrid of the less-sharp cloud lands in mvg_corner (with its own
  // scratch, the chain may run on a second stream), that of the less-flat cloud in lf_raw (free once the per-ring VoxelGrid has read it)
  DevBuf mvg, vg_scratch2;
  float4* mvg_corner = nullptr;
};

static int spin_key_bits(int m) { int b = 0; while ((1 << b) < m) b++; return 32 + b; }

struct SpinFilter {
  float thr2;
  __device__ __forceinline__ bool operator()(const float4& p) const {
    if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) return false;
    if (fabsf(p.x) > SPIN_MAX_COORD || fabsf(p.y) > SPIN_MAX_COORD || fabsf(p.z) > SPIN_MAX_COORD) return false;
    return !(p.x * p.x + p.y * p.y + p.z * p.z < thr2);
  }
};

// ring (scanID) of a point, -1 when the reference drops it (:430-460)
__device__ __forceinline__ int spin_ring(float x, float y, float z, int rings) {
  const float t = (float)atan((double)(z / sqrtf(x * x + y * y)));
  const float angle = (float)((double)(t * 180.0f) / SPIN_PI);
  if (rings == 16) {
    const int id = (int)((double)((angle + 15.0f) / 2.0f) + 0.5);
    return (id > 15 || id < 0) ? -1 : id;
  }
  int id;
  if ((double)angle >= -8.83) id = (int)((double)(2.0f - angle) * 3.0 + 0.5);
  else id = 32 + (int)((-8.83 - (double)angle) * 2.0 + 0.5);
  if (angle > 2.0f || (double)angle < -24.33 || id > 50 || id < 0) return -1;
  return id;
}
__device__ __forceinline__ float spin_ori(float x, float y) { return -(float)atan2((double)y, (double)x); }
__device__ __forceinline__ void spin_start_end(const float4* f, int nf, float& so, float& eo) {
  so = spin_ori(f[0].x, f[0].y);
  eo = (float)((double)spin_ori(f[nf - 1].x, f[nf - 1].y) + 2 * SPIN_PI);
  if ((double)(eo - so) > 3 * SPIN_PI) eo = (float)((double)eo - 2 * SPIN_PI);
  else if ((double)(eo - so) < SPIN_PI) eo = (float)((double)eo + 2 * SPIN_PI);
}
__device__ __forceinline__ float spin_first_branch(float ori, float so) {
  if ((double)ori < (double)so - SPIN_PI / 2) ori = (float)((double)ori + 2 * SPIN_PI);
  else if ((double)ori > (double)so + SPIN_PI * 3 / 2) ori = (float)((double)ori - 2 * SPIN_PI);
  return ori;
}

// ring id as the bucket key (dropped and padding points: past every ring), first-branch halfPassed test
__global__ void spin_ring_kernel(const float4* __restrict__ f, int n, SpinMeta* __restrict__ m, int rings, int* __restrict__ key, int* __restrict__ val) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const int nf = m->nf;
  int r = -1;
  if (k < nf) {
    const float4 p = f[k];
    r = spin_ring(p.x, p.y, p.z, rings);
    if (r >= 0) {
      atomicAdd(&m->ring_cnt[r], 1);
      float so, eo; spin_start_end(f, nf, so, eo);
      const float ori = spin_first_branch(spin_ori(p.x, p.y), so);
      if ((double)(ori - so) > SPIN_PI) atomicMin(&m->first_half, k);
    }
  }
  key[k] = r < 0 ? SPIN_MAX_RINGS : r;
  val[k] = k;
}

// ring offsets, N, scanStartInd / scanEndInd and the sub-scan bounds (:513-521, :638-640); one thread per ring
__global__ void spin_layout_kernel(SpinMeta* __restrict__ m, int rings) {
  __shared__ int begin[SPIN_MAX_RINGS + 1];
  if (threadIdx.x == 0) {
    int s = 0;
    for (int r = 0; r < rings; r++) { begin[r] = s; s += m->ring_cnt[r]; }
    begin[rings] = s;
    m->counts[0] = s;
  }
  __syncthreads();
  const int r = threadIdx.x;
  if (r > rings) return;
  m->ring_begin[r] = begin[r];
  if (r == rings) return;
  const int S = begin[r] + 5, E = begin[r + 1] - 6;
  for (int j = 0; j < SPIN_SUB; j++) {
    m->sp[r * SPIN_SUB + j] = (S * (6 - j) + E * j) / 6;
    m->ep[r * SPIN_SUB + j] = (S * (5 - j) + E * (j + 1)) / 6 - 1;
  }
}

// the ring-ordered cloud with intensity = ring + 0.1 relTime (:469-503)
__global__ void spin_gather_kernel(const float4* __restrict__ f, const int* __restrict__ key, const int* __restrict__ val, const SpinMeta* __restrict__ m, int n,
                                   float4* __restrict__ cloud) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n || j >= m->counts[0]) return;
  const int k = val[j], r = key[j];
  const float4 p = f[k];
  float so, eo; spin_start_end(f, m->nf, so, eo);
  float ori = spin_ori(p.x, p.y);
  if (k <= m->first_half) {
    ori = spin_first_branch(ori, so);
  } else {
    ori = (float)((double)ori + 2 * SPIN_PI);
    if ((double)ori < (double)eo - SPIN_PI * 3 / 2) ori = (float)((double)ori + 2 * SPIN_PI);
    else if ((double)ori > (double)eo + SPIN_PI / 2) ori = (float)((double)ori - 2 * SPIN_PI);
  }
  const float rel = (ori - so) / (eo - so);
  cloud[j] = make_float4(p.x, p.y, p.z, (float)((double)r + 0.1 * (double)rel));
}

// curvature, backward occlusion, parallel beam (:524-598) for i in [5, N-5); the gap cuts for i in [1, N)
__global__ void spin_curv_kernel(const float4* __restrict__ c, const SpinMeta* __restrict__ m, int n, float* __restrict__ curv, unsigned char* __restrict__ occl,
                                 unsigned char* __restrict__ beam, unsigned* __restrict__ cut) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int N = m->counts[0];
  bool gap = false;
  if (i < N) {
    float cv = 0.f; unsigned char oc = 0, bm = 0;
    const float4 p = c[i];
    if (i >= 5 && i < N - 5) {
      float dx = c[i - 5].x + c[i - 4].x + c[i - 3].x + c[i - 2].x + c[i - 1].x - 10 * p.x + c[i + 1].x + c[i + 2].x + c[i + 3].x + c[i + 4].x + c[i + 5].x;
      float dy = c[i - 5].y + c[i - 4].y + c[i - 3].y + c[i - 2].y + c[i - 1].y - 10 * p.y + c[i + 1].y + c[i + 2].y + c[i + 3].y + c[i + 4].y + c[i + 5].y;
      float dz = c[i - 5].z + c[i - 4].z + c[i - 3].z + c[i - 2].z + c[i - 1].z - 10 * p.z + c[i + 1].z + c[i + 2].z + c[i + 3].z + c[i + 4].z + c[i + 5].z;
      const float diff = dx * dx + dy * dy + dz * dz;
      cv = diff;
      if ((double)diff > 0.1) {
        const float4 q = c[i + 1];
        const float depth1 = sqrtf(p.x * p.x + p.y * p.y + p.z * p.z);
        const float depth2 = sqrtf(q.x * q.x + q.y * q.y + q.z * q.z);
        if (depth1 > depth2) {
          dx = q.x - p.x * depth2 / depth1; dy = q.y - p.y * depth2 / depth1; dz = q.z - p.z * depth2 / depth1;
          if ((double)(sqrtf(dx * dx + dy * dy + dz * dz) / depth2) < 0.1) oc = 1;   // marks i-5 ... i
        }
        // the forward marks (depth1 <= depth2) are reset by the later iterations (:533) and never survive
      }
      const float4 o = c[i - 1];
      const float dx2 = p.x - o.x, dy2 = p.y - o.y, dz2 = p.z - o.z;
      const float diff2 = dx2 * dx2 + dy2 * dy2 + dz2 * dz2;
      const float dis = p.x * p.x + p.y * p.y + p.z * p.z;
      if ((double)diff > 0.0002 * (double)dis && (double)diff2 > 0.0002 * (double)dis) bm = 1;
    }
    curv[i] = cv; occl[i] = oc; beam[i] = bm;
    if (i >= 1) {
      const float4 o = c[i - 1];
      const float gx = p.x - o.x, gy = p.y - o.y, gz = p.z - o.z;
      gap = (double)(gx * gx + gy * gy + gz * gz) > 0.05;
    }
  }
  const unsigned b = __ballot_sync(FULL, gap);
  if ((threadIdx.x & 31) == 0 && i - (int)(threadIdx.x & 31) < n) cut[i >> 5] = b;
}

// sub-scan of index i (-1: none), from the ring offsets and the sub-scan bounds
__device__ __forceinline__ int spin_sub_of(const SpinMeta* m, int rings, int i) {
  int lo = 0, hi = rings;   // last ring with begin <= i
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (m->ring_begin[mid] <= i) lo = mid; else hi = mid; }
  for (int j = 0; j < SPIN_SUB; j++) { const int g = lo * SPIN_SUB + j; if (i >= m->sp[g] && i <= m->ep[g]) return g; }
  return -1;
}
// picked before the selection: beam(k) OR any backward occlusion of i = k ... min(k + 5, N - 6); the sort keys; labels cleared
__global__ void spin_flags_kernel(const float* __restrict__ curv, const unsigned char* __restrict__ occl, const unsigned char* __restrict__ beam, const SpinMeta* __restrict__ m,
                                  int n, int rings, unsigned* __restrict__ picked, unsigned* __restrict__ picked0, unsigned long long* __restrict__ key, int* __restrict__ val,
                                  signed char* __restrict__ label, short* __restrict__ sid) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int N = m->counts[0];
  bool pk = false;
  if (i < N) {
    if (i >= 5 && i < N - 5) {
      pk = beam[i] != 0;
      for (int t = i; t <= i + 5 && t <= N - 6; t++) pk = pk || occl[t] != 0;
    }
    const int g = spin_sub_of(m, rings, i);
    sid[i] = (short)g;
    label[i] = 0;
    key[i] = ((unsigned long long)(unsigned)(g >= 0 ? m->sp[g] : i) << 32) | (unsigned long long)__float_as_uint(curv[i]);
    val[i] = i;
  } else if (i < n) {
    key[i] = ~0ull; val[i] = i;
  }
  const unsigned b = __ballot_sync(FULL, pk);
  if ((threadIdx.x & 31) == 0 && i - (int)(threadIdx.x & 31) < n) { picked[i >> 5] = b; picked0[i >> 5] = b; }
}

// chains: a new chain starts at a non-empty sub-scan when a cut lies in (ep of the previous non-empty sub-scan, its sp]
__device__ __forceinline__ bool spin_cut(const unsigned* cut, int k) { return (cut[k >> 5] >> (k & 31)) & 1u; }
__global__ void spin_chains_kernel(const unsigned* __restrict__ cut, SpinMeta* __restrict__ m, int rings) {
  if (threadIdx.x != 0) return;
  const int G = rings * SPIN_SUB;
  int prev = -1, nch = 0, first_sp = 0, longest = 0;
  for (int g = 0; g < G; g++) {
    const int s = m->sp[g], e = m->ep[g];
    if (e < s) continue;
    bool brk = prev < 0;
    for (int k = prev + 1; !brk && k <= s; k++) brk = spin_cut(cut, k);
    if (brk) {
      if (nch) longest = max(longest, prev - first_sp + 1);
      m->chain_first[nch++] = g; first_sp = s;
    }
    prev = e;
  }
  if (nch) longest = max(longest, prev - first_sp + 1);
  m->chain_first[nch] = G;
  m->counts[5] = nch; m->counts[6] = longest;
}

// walks of a pick at ind (:687-710, :733-756): the run up to the first cut, at most cap points, inside [0, N)
__device__ __forceinline__ int spin_reach_right(const unsigned* cut, int ind, int cap, int N) {
  const int lim = min(cap, N - 1 - ind);   // marks ind + 1 ... ind + r
  int r = 0;
  while (r < lim) {
    const int k = ind + r + 1;
    const unsigned w = __ldg(&cut[k >> 5]) >> (k & 31);
    if (w) { r += __ffs(w) - 1; return min(r, lim); }
    r += 32 - (k & 31);
  }
  return lim;
}
__device__ __forceinline__ int spin_reach_left(const unsigned* cut, int ind, int cap) {
  const int lim = min(cap, ind);   // marks ind - 1 ... ind - l; stops at the first k <= ind with a cut (the gap between k - 1 and k)
  int l = 0;
  while (l < lim) {
    const int k = ind - l;         // next gap to test: between k - 1 and k
    const unsigned w = __ldg(&cut[k >> 5]) << (31 - (k & 31));
    if (w) { l += __clz(w); return min(l, lim); }
    l += (k & 31) + 1;
  }
  return lim;
}
__device__ __forceinline__ void spin_mark(unsigned* picked, int lo, int hi, int lane) {
  const int wlo = lo >> 5, whi = hi >> 5;
  for (int w = wlo + lane; w <= whi; w += 32) {
    unsigned mask = FULL;
    if (w == wlo) mask &= FULL << (lo & 31);
    if (w == whi) mask &= FULL >> (31 - (hi & 31));
    atomicOr(&picked[w], mask);
  }
}
__device__ __forceinline__ bool spin_picked(const unsigned* picked, int k) { return (__ldcg(&picked[k >> 5]) >> (k & 31)) & 1u; }

// The selection (:656-758), one warp per chain.  Candidates are visited 32 at a time in sorted order; the first eligible lane is the next pick,
// its interval is marked with whole-word atomics, then eligibility is re-read.  Picks go to per-sub-scan slots (output order = sub-scan order).
#define SPIN_SELECT_WARPS 4
__global__ void __launch_bounds__(SPIN_SELECT_WARPS * 32) spin_select_kernel(const float* __restrict__ curv, const int* __restrict__ sorted, const unsigned* __restrict__ cut,
                                                                             SpinMeta* __restrict__ m, unsigned* __restrict__ picked, signed char* __restrict__ label,
                                                                             int* __restrict__ sharp_idx, int* __restrict__ flat_idx) {
  const int w = blockIdx.x * SPIN_SELECT_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= m->counts[5]) return;
  const int N = m->counts[0];
  for (int g = m->chain_first[w]; g < m->chain_first[w + 1]; g++) {
    const int s = m->sp[g], e = m->ep[g];
    if (e < s) continue;
    // sharp: descending curvature, > 0.5 (sharp_point_threshold * 10 in float)
    int cnt = 0; bool stop = false;
    for (int base = e; base >= s && !stop; base -= 32) {
      const int pos = base - lane;
      const bool valid = pos >= s;
      const int ind = valid ? sorted[pos] : 0;
      const bool cand = valid && curv[ind] > 0.05f * 10;
      if (__ballot_sync(FULL, !cand)) stop = true;   // sorted: every later candidate fails as well
      bool elig = cand && !spin_picked(picked, ind);
      unsigned bal = __ballot_sync(FULL, elig);
      while (bal) {
        const int f = __ffs(bal) - 1;
        const int pi = __shfl_sync(FULL, ind, f);
        if (++cnt > SPIN_SHARP_MAX) { stop = true; break; }
        if (lane == 0) { sharp_idx[g * SPIN_SHARP_MAX + cnt - 1] = pi; label[pi] = cnt <= 20 ? 2 : 1; }
        spin_mark(picked, pi - spin_reach_left(cut, pi, 500), pi + spin_reach_right(cut, pi, 500, N), lane);
        __syncwarp();
        elig = elig && !spin_picked(picked, ind);
        bal = __ballot_sync(FULL, elig);
      }
    }
    // flat: ascending curvature, < 0.05; the 5th pick ends the pass before it marks anything
    int fc = 0; stop = false;
    for (int base = s; base <= e && !stop; base += 32) {
      const int pos = base + lane;
      const bool valid = pos <= e;
      const int ind = valid ? sorted[pos] : 0;
      const bool cand = valid && curv[ind] < 0.05f;
      if (__ballot_sync(FULL, !cand)) stop = true;
      bool elig = cand && !spin_picked(picked, ind);
      unsigned bal = __ballot_sync(FULL, elig);
      while (bal) {
        const int f = __ffs(bal) - 1;
        const int pi = __shfl_sync(FULL, ind, f);
        if (lane == 0) { flat_idx[g * SPIN_FLAT_MAX + fc] = pi; label[pi] = -1; }
        if (++fc >= SPIN_FLAT_MAX) { stop = true; break; }
        spin_mark(picked, pi - spin_reach_left(cut, pi, 5), pi + spin_reach_right(cut, pi, 5, N), lane);
        __syncwarp();
        elig = elig && !spin_picked(picked, ind);
        bal = __ballot_sync(FULL, elig);
      }
    }
    if (lane == 0) { m->nsharp[g] = min(cnt, SPIN_SHARP_MAX); m->nflat[g] = fc; }
    __syncwarp();
  }
}

// less flat: the sub-scan points with label <= 0 (:761-767), counted per ring
__global__ void spin_lessflat_kernel(const signed char* __restrict__ label, const short* __restrict__ sid, SpinMeta* __restrict__ m, int n, unsigned char* __restrict__ flag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  bool f = false;
  if (i < m->counts[0]) {
    const int g = sid[i];
    f = g >= 0 && label[i] <= 0;
    if (f) atomicAdd(&m->lf_cnt[g / SPIN_SUB], 1);
  }
  flag[i] = f;
}

// the sharp / less sharp / flat clouds in push order (sub-scan order, pick order inside), the ring ends of the less-flat cloud, the counts
__global__ void spin_out_kernel(const float4* __restrict__ cloud, SpinMeta* __restrict__ m, int rings, const int* __restrict__ sharp_idx, const int* __restrict__ flat_idx,
                                float4* __restrict__ o_sharp, float4* __restrict__ o_less, float4* __restrict__ o_flat) {
  __shared__ int off[3][SPIN_MAX_SUBS + 1];
  const int G = rings * SPIN_SUB;
  if (threadIdx.x == 0) {
    int a = 0, b = 0, c = 0;
    for (int g = 0; g < G; g++) { off[0][g] = a; off[1][g] = b; off[2][g] = c; a += min(m->nsharp[g], 20); b += m->nsharp[g]; c += m->nflat[g]; }
    off[0][G] = a; off[1][G] = b; off[2][G] = c;
    m->counts[1] = a; m->counts[2] = b; m->counts[3] = c;
    int e = 0;
    for (int r = 0; r < rings; r++) { e += m->lf_cnt[r]; m->lf_end[r] = e; }
    m->counts[7] = e;
  }
  __syncthreads();
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    const int ns = m->nsharp[g], nfl = m->nflat[g];
    for (int j = 0; j < ns; j++) {
      const float4 p = cloud[sharp_idx[g * SPIN_SHARP_MAX + j]];
      if (j < 20) o_sharp[off[0][g] + j] = p;
      o_less[off[1][g] + j] = p;
    }
    for (int j = 0; j < nfl; j++) o_flat[off[2][g] + j] = cloud[flat_idx[g * SPIN_FLAT_MAX + j]];
  }
}
__global__ void spin_final_kernel(SpinMeta* __restrict__ m, int rings) { m->counts[4] = m->vg_end[rings - 1]; }

// The streaming mapper's max_t: the largest intensity (ring + 0.1 relTime) of the full cloud, from find_min_max_intensity's start value -10000
// (laser_mapping.hpp:1243-1253, :1336-1347).  One block; the intensities are finite, so the order-preserving int max is the float max.
#define SPIN_MAXT_THREADS 1024
__global__ void __launch_bounds__(SPIN_MAXT_THREADS) spin_max_t_kernel(const float4* __restrict__ cloud, SpinMeta* __restrict__ m) {
  __shared__ int wmax[SPIN_MAXT_THREADS / 32];
  const int N = m->counts[0];
  int mx = ll_f2ord(-10000.0f);
  for (int i = threadIdx.x; i < N; i += SPIN_MAXT_THREADS) mx = max(mx, ll_f2ord(cloud[i].w));
  mx = __reduce_max_sync(FULL, mx);
  if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x < 32) {
    mx = __reduce_max_sync(FULL, wmax[threadIdx.x]);
    if (threadIdx.x == 0) m->feat[2] = mx;
  }
}

// ------------------------------------------------------------------------------------------------------------------------------------------ host
static void spin_layout(ll_spin* h, Carve& c) {
  const int M = h->cfg.max_points, G = h->rings * SPIN_SUB;
  h->in4 = c.take<float4>(M); h->filt = c.take<float4>(M); h->cloud = c.take<float4>(M);
  for (int k = 0; k < 2; k++) { h->rkey[k] = c.take<int>(M); h->rval[k] = c.take<int>(M); h->ckey[k] = c.take<unsigned long long>(M); h->cval[k] = c.take<int>(M); }
  h->curv = c.take<float>(M); h->occl = c.take<unsigned char>(M); h->beam = c.take<unsigned char>(M);
  const int W = M / 32 + 2;
  h->picked = c.take<unsigned>(W); h->picked0 = c.take<unsigned>(W); h->cut = c.take<unsigned>(W);
  h->label = c.take<signed char>(M); h->sid = c.take<short>(M); h->lfflag = c.take<unsigned char>(M);
  h->sharp_idx = c.take<int>((size_t)G * SPIN_SHARP_MAX); h->flat_idx = c.take<int>((size_t)G * SPIN_FLAT_MAX);
  h->out_sharp = c.take<float4>(std::min(M, G * 20)); h->out_less_sharp = c.take<float4>(std::min(M, G * SPIN_SHARP_MAX));
  h->out_flat = c.take<float4>(std::min(M, G * SPIN_FLAT_MAX));
  h->lf_raw = c.take<float4>(M); h->out_less_flat = c.take<float4>(M);
  h->meta = c.take<SpinMeta>(1);
  h->tmp = c.take<char>(h->tmp_bytes);
}
static int spin_corner_cap(const ll_spin* h) { return std::min(h->cfg.max_points, h->rings * SPIN_SUB * SPIN_SHARP_MAX); }   // out_less_sharp's size
static size_t spin_tmp_bytes(int M) {
  size_t a = 0, b = 0, d = 0, e = 0;
  cub::DeviceSelect::If(nullptr, a, (float4*)nullptr, (float4*)nullptr, (int*)nullptr, M, SpinFilter{0.f});
  cub::DeviceRadixSort::SortPairs(nullptr, b, (int*)nullptr, (int*)nullptr, (int*)nullptr, (int*)nullptr, M, 0, 7);
  cub::DeviceRadixSort::SortPairs(nullptr, d, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int*)nullptr, (int*)nullptr, M, 0, spin_key_bits(M));
  cub::DeviceSelect::Flagged(nullptr, e, (float4*)nullptr, (unsigned char*)nullptr, (float4*)nullptr, (int*)nullptr, M);
  return std::max(std::max(a, b), std::max(d, e));
}

// The front end on the streams fs (the extraction on fs.main).  mapping == null (ll_spin_extract): the counts read back with one synchronisation.
// Otherwise (the streaming mapper's sweep) also the mapping node's input VoxelGrids (laser_mapping.hpp:1367-1373) on the device counts of the
// less-sharp and less-flat clouds, one stage per chain, and max_t; SpinMeta::counts and ::feat land in the pinned block, without a
// synchronisation (spin_sweep_finish reads them once the work has completed).
static int spin_run(ll_spin* h, const FrontStreams& fs, const void* raw, size_t n_, int fmt, int where, const ll_pipeline_cfg* mapping) {
  ll_ctx* ctx = h->ctx;
  cudaStream_t s = fs.main;
  const int n = (int)n_, R = h->rings, G = R * SPIN_SUB, B = 256, nb = ll_div_up(n, B);
  SpinMeta* m = h->meta;
  LL_CUDA(ctx, cudaMemsetAsync(m, 0, sizeof(SpinMeta), s));
  LL_CUDA(ctx, cudaMemsetAsync(&m->first_half, 0x7f, sizeof(int), s));
  LL_TRY(upload_cloud(ctx, s, raw, n_, fmt, where, h->in4));
  const float thr = h->cfg.minimum_range;
  size_t tb = h->tmp_bytes;
  LL_CUDA(ctx, cub::DeviceSelect::If(h->tmp, tb, h->in4, h->filt, &m->nf, n, SpinFilter{thr * thr}, s));
  spin_ring_kernel<<<nb, B, 0, s>>>(h->filt, n, m, R, h->rkey[0], h->rval[0]);
  tb = h->tmp_bytes;
  LL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(h->tmp, tb, h->rkey[0], h->rkey[1], h->rval[0], h->rval[1], n, 0, 7, s));
  spin_layout_kernel<<<1, SPIN_MAX_RINGS + 1, 0, s>>>(m, R);
  spin_gather_kernel<<<nb, B, 0, s>>>(h->filt, h->rkey[1], h->rval[1], m, n, h->cloud);
  spin_curv_kernel<<<nb, B, 0, s>>>(h->cloud, m, n, h->curv, h->occl, h->beam, h->cut);
  spin_flags_kernel<<<nb, B, 0, s>>>(h->curv, h->occl, h->beam, m, n, R, h->picked, h->picked0, h->ckey[0], h->cval[0], h->label, h->sid);
  tb = h->tmp_bytes;
  LL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(h->tmp, tb, h->ckey[0], h->ckey[1], h->cval[0], h->cval[1], n, 0, spin_key_bits(h->cfg.max_points), s));
  spin_chains_kernel<<<1, 32, 0, s>>>(h->cut, m, R);
  spin_select_kernel<<<ll_div_up(G, SPIN_SELECT_WARPS), SPIN_SELECT_WARPS * 32, 0, s>>>(h->curv, h->cval[1], h->cut, m, h->picked, h->label, h->sharp_idx, h->flat_idx);
  spin_lessflat_kernel<<<nb, B, 0, s>>>(h->label, h->sid, m, n, h->lfflag);
  tb = h->tmp_bytes;
  LL_CUDA(ctx, cub::DeviceSelect::Flagged(h->tmp, tb, h->cloud, h->lfflag, h->lf_raw, &m->nlf, n, s));
  spin_out_kernel<<<1, 128, 0, s>>>(h->cloud, m, R, h->sharp_idx, h->flat_idx, h->out_sharp, h->out_less_sharp, h->out_flat);
  LL_TRY(launch_voxel_grid_segments(ctx, s, h->vg_scratch, h->lf_raw, n, m->lf_end, R, h->cfg.plane_resolution / 2, h->out_less_flat, m->vg_end));
  spin_final_kernel<<<1, 1, 0, s>>>(m, R);
  // select (2), ring sort (histogram, scan, 1 pass), curvature sort (histogram, scan, one pass per 8 key bits), flagged select (2), 10 kernels
  ctx->launches += 2 + 3 + 2 + (uint64_t)(spin_key_bits(h->cfg.max_points) + 7) / 8 + 2 + 10;
  LL_CUDA(ctx, cudaGetLastError());
  if (!mapping) {
    LL_CUDA(ctx, cudaMemcpyAsync(h->pin, m->counts, sizeof(m->counts), cudaMemcpyDeviceToHost, s));
    LL_CUDA(ctx, cudaStreamSynchronize(s));
    return LL_OK;
  }
  // less sharp -> corners at mapping_leaf_corner, less flat -> surfaces at mapping_leaf_surf (the remapped /pc2_corners and /pc2_surface)
  const VgChain c[2] = {
      {{h->out_less_sharp, std::min(n, spin_corner_cap(h)), &m->counts[2], 1, {mapping->mapping_leaf_corner, 0.f}, {h->mvg_corner, nullptr}, {&m->feat[0], nullptr}},
       &h->vg_scratch2, fs.corner},
      {{h->out_less_flat, n, &m->counts[4], 1, {mapping->mapping_leaf_surf, 0.f}, {h->lf_raw, nullptr}, {&m->feat[1], nullptr}}, &h->vg_scratch, fs.main}};
  LL_TRY(launch_voxel_chains(ctx, s, c, 2, fs.fork, fs.join));
  spin_max_t_kernel<<<1, SPIN_MAXT_THREADS, 0, s>>>(h->cloud, m); ctx->launches++;
  LL_CUDA(ctx, cudaGetLastError());
  static_assert(offsetof(SpinMeta, feat) == offsetof(SpinMeta, counts) + sizeof(SpinMeta::counts), "counts and feat are read back together");
  LL_CUDA(ctx, cudaMemcpyAsync(h->pin, m->counts, sizeof(m->counts) + sizeof(m->feat), cudaMemcpyDeviceToHost, s));
  return LL_OK;
}

// ------------------------------------------------------------------------------------------------------ the streaming mapper's sweeps
ll_ctx* spin_ctx(const ll_spin* h) { return h->ctx; }
size_t spin_max_points(const ll_spin* h) { return (size_t)h->cfg.max_points; }

int spin_sweep_enqueue(ll_spin* h, const FrontStreams& fs, const void* raw, size_t n, int fmt, int where, const ll_pipeline_cfg* pc) {
  if (n == 0) {   // no front end: the counts of an empty sweep (the pinned block is free, the previous sweep's finish has read it), and the
                  // device count of the full cloud that loop_sweep_cloud hands on, in stream order behind the previous sweep's copy (fe_free)
    for (int k = 0; k < 12; k++) h->pin[k] = 0;
    h->pin[10] = ll_f2ord(-10000.0f);
    LL_CUDA(h->ctx, cudaMemsetAsync(&h->meta->counts[0], 0, sizeof(int), fs.main));
    return LL_OK;
  }
  return spin_run(h, fs, raw, n, fmt, where, pc);
}

void spin_sweep_finish(ll_spin* h, size_t n, const float4** corner, int* nc, const float4** surf, int* ns, float* max_t) {
  for (int k = 0; k < 8; k++) h->last_counts[k] = h->pin[k];
  h->extracted = 1; h->last_n = (int)n;
  *corner = h->mvg_corner; *nc = h->pin[8]; *surf = h->lf_raw; *ns = h->pin[9]; *max_t = ll_ord2f(h->pin[10]);
}

const float4* spin_full_cloud(const ll_spin* h, int* n, const int** d_n) { *n = h->last_counts[0]; *d_n = &h->meta->counts[0]; return h->cloud; }
void spin_forget(ll_spin* h) { h->extracted = 0; }

extern "C" {

void ll_spin_cfg_default(ll_spin_cfg* c) {
  if (!c) return;
  c->scan_line = 16;            // feature_extraction/scan_line (:137)
  c->minimum_range = 0.1f;      // feature_extraction/minimum_range (:140)
  c->plane_resolution = 0.4f;   // feature_extraction/mapping_plane_resolution of the shipped YAMLs (VoxelGrid leaf 0.2, :192)
  c->max_points = 400000;       // m_pc_curvature and the other per-point arrays (:75-78)
}

int ll_spin_create(ll_ctx* ctx, const ll_spin_cfg* cfg, ll_spin** out) {
  if (!ctx || !cfg || !out) return LL_ERR_INVALID;
  if (cfg->scan_line != 16 && cfg->scan_line != 64) { ctx->set_error("scan_line must be 16 or 64 (laser_feature_extractor.hpp:160-164)"); return LL_ERR_INVALID; }
  if (cfg->max_points < 1 || cfg->max_points > (1 << 24) || !(cfg->minimum_range >= 0.f) || !std::isfinite(cfg->minimum_range) || !(cfg->plane_resolution > 0.f) ||
      !std::isfinite(cfg->plane_resolution)) { ctx->set_error("ll_spin_cfg: max_points outside 1 ... 2^24 or a non-finite / non-positive resolution"); return LL_ERR_INVALID; }
  cudaSetDevice(ctx->device);
  ll_spin* h = new ll_spin();
  h->ctx = ctx; h->cfg = *cfg; h->rings = cfg->scan_line;
  h->tmp_bytes = spin_tmp_bytes(cfg->max_points);
  cudaError_t e = h->arena.carve([&](Carve& c) { spin_layout(h, c); });
  if (e == cudaSuccess) e = h->vg_scratch.reserve(std::max(voxel_grid_bytes(cfg->max_points, h->rings), voxel_grid_bytes(cfg->max_points)));
  if (e == cudaSuccess) e = h->mvg.carve([&](Carve& c) { h->mvg_corner = c.take<float4>(spin_corner_cap(h)); });
  if (e == cudaSuccess) e = h->vg_scratch2.reserve(voxel_grid_bytes(spin_corner_cap(h)));
  if (e == cudaSuccess) e = cudaMallocHost((void**)&h->pin, sizeof(SpinMeta::counts) + sizeof(SpinMeta::feat));
  if (e != cudaSuccess) { ctx->set_error(std::string("ll_spin_create: ") + cudaGetErrorString(e)); ll_spin_release(h); return LL_ERR_CUDA; }
  *out = h; return LL_OK;
}

void ll_spin_release(ll_spin* h) {
  if (!h) return;
  cudaSetDevice(h->ctx->device);
  h->arena.release(); h->vg_scratch.release(); h->mvg.release(); h->vg_scratch2.release();
  if (h->pin) cudaFreeHost(h->pin);
  delete h;
}

int ll_spin_extract(ll_spin* h, const void* raw, size_t n, int fmt, int where, size_t counts[5]) {
  if (!h) return LL_ERR_INVALID;
  ll_ctx* ctx = h->ctx;
  if ((n > 0 && !raw) || (where != LL_HOST && where != LL_DEVICE) || (fmt != LL_FMT_XYZI16 && fmt != LL_FMT_PCL32 && fmt != LL_FMT_STRIDED)) {
    ctx->set_error("ll_spin_extract: null input, unknown fmt or where"); return LL_ERR_INVALID;
  }
  if (n > (size_t)h->cfg.max_points) { ctx->set_error("ll_spin_extract: more points than ll_spin_cfg::max_points"); return LL_ERR_CAPACITY; }
  cudaSetDevice(ctx->device);
  h->extracted = 0;
  if (n == 0) { for (int k = 0; k < 8; k++) h->last_counts[k] = 0; }
  else { LL_TRY(spin_run(h, ctx->own_front(), raw, n, fmt, where, nullptr)); for (int k = 0; k < 8; k++) h->last_counts[k] = h->pin[k]; }
  h->extracted = 1; h->last_n = (int)n;
  if (counts) for (int k = 0; k < 5; k++) counts[k] = (size_t)h->last_counts[k];
  return LL_OK;
}

int ll_spin_cloud(ll_spin* h, int which, ll_point* out_host, size_t cap, size_t* n_out, const ll_point** out_dev) {
  if (!h || !n_out || which < LL_SPIN_FULL || which > LL_SPIN_LESS_FLAT) return LL_ERR_INVALID;
  if (!h->extracted) { h->ctx->set_error("ll_spin_cloud: nothing extracted"); return LL_ERR_INVALID; }
  const float4* src[5] = {h->cloud, h->out_sharp, h->out_less_sharp, h->out_flat, h->out_less_flat};
  const size_t n = (size_t)h->last_counts[which];
  *n_out = n;
  const ll_point* d = n ? (const ll_point*)src[which] : nullptr;
  if (out_dev) *out_dev = d;
  if (out_host && n) {
    ll_ctx* ctx = h->ctx;
    cudaSetDevice(ctx->device);
    LL_CUDA(ctx, cudaMemcpyAsync(out_host, d, (n < cap ? n : cap) * 16, cudaMemcpyDeviceToHost, ctx->stream));
    LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  return LL_OK;
}

int ll_spin_point_info(ll_spin* h, int32_t* ring, float* curvature, int32_t* picked, int32_t* label, size_t cap, size_t* n_out) {
  if (!h || !n_out) return LL_ERR_INVALID;
  if (!h->extracted) { h->ctx->set_error("ll_spin_point_info: nothing extracted"); return LL_ERR_INVALID; }
  ll_ctx* ctx = h->ctx;
  const size_t N = (size_t)h->last_counts[0], k = N < cap ? N : cap;
  *n_out = N;
  if (k == 0) return LL_OK;
  cudaSetDevice(ctx->device);
  cudaStream_t s = ctx->stream;
  int begin[SPIN_MAX_RINGS + 1];
  std::vector<unsigned> p(picked ? k / 32 + 1 : 0);
  std::vector<signed char> l(label ? k : 0);
  LL_CUDA(ctx, cudaMemcpyAsync(begin, h->meta->ring_begin, sizeof(begin), cudaMemcpyDeviceToHost, s));
  if (curvature) LL_CUDA(ctx, cudaMemcpyAsync(curvature, h->curv, k * 4, cudaMemcpyDeviceToHost, s));
  if (picked) LL_CUDA(ctx, cudaMemcpyAsync(p.data(), h->picked0, (k / 32 + 1) * 4, cudaMemcpyDeviceToHost, s));
  if (label) LL_CUDA(ctx, cudaMemcpyAsync(l.data(), h->label, k, cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  int r = 0;
  for (size_t i = 0; i < k; i++) {
    while (r + 1 < h->rings && begin[r + 1] <= (int)i) r++;
    if (ring) ring[i] = r;
    if (picked) picked[i] = (p[i >> 5] >> (i & 31)) & 1u;
    if (label) label[i] = l[i];
  }
  return LL_OK;
}

int ll_spin_chains(const ll_spin* h, int* n_chains, int* longest) {
  if (!h || !h->extracted) return LL_ERR_INVALID;
  if (n_chains) *n_chains = h->last_counts[5];
  if (longest) *longest = h->last_counts[6];
  return LL_OK;
}

}  // extern "C"
