// Loop detection on the device: keyframes over a full-resolution cell map, their feature images and the candidate search.
//
// Replaces, on the reference side:
//   append_cloud(full, &cell_vec) + Maps_keyframe::add_cells     laser_mapping.hpp:1527-1533, cell_map_keyframe.hpp:585-665,1243-1261
//   Points_cloud_cell mean / covariance / determine_feature       cell_map_keyframe.hpp:215-315,378-419,436-473
//   Maps_keyframe::analyze (centre, ROI range, feature images)   cell_map_keyframe.hpp:1231-1241,1292-1319,1358-1494,1554-1567
//   extract_specify_points / get_all_pointcloud                    cell_map_keyframe.hpp:1263-1290
//   the similarity gates of service_loop_detection                 laser_mapping.hpp:988-1033, cell_map_keyframe.hpp:1144-1229,1321-1356
//
// A keyframe cell is one incarnation of a map cell: (cell slot, epoch).  A revisit starts a new epoch in the map (a new Points_cloud_cell in the
// reference), the old incarnation keeps its points in the store, so a keyframe that holds it still sees exactly the points it had.  A keyframe's
// cells are kept sorted by (cell key, epoch): ascending (k, j, i), the order the cell map already visits cells in; it is the order of every
// order-sensitive sum and of the typed clouds.  Points inside a cell are in append order.
// Compiled with -fmad=false: the per-cell float sums, the centre and the images round like the oracle's scalar code.
#include <cub/cub.cuh>
#include <cmath>
#include "common.cuh"
#include "kernels.cuh"
#include "cellmap.cuh"

#define KF_RES 60                      // PHI_RESOLUTION = THETA_RESOLUTION (cell_map_keyframe.hpp:35-36)
#define KF_PIX (KF_RES * KF_RES)
#define KF_PAD 30                      // add_padding_to_feature_image(img_b, PHI_RESOLUTION * 0.5, THETA_RESOLUTION * 0.5)
#define KF_PW (KF_RES + 2 * KF_PAD)    // 120
#define KF_POS (2 * KF_PAD + 1)        // 61 x 61 template positions
#define KF_SEARCH_THREADS 256
#define KF_STALE "the cell map's store was rebuilt (down-sample-and-replace assembly or image load) after this keyframe took its cells"

struct ll_keyframe {
  int device = 0;
  const ll_cellmap* map = nullptr;     // the cell map its cells belong to (set by the first append)
  int generation = 0;                  // the map's store generation its (slot, epoch) pairs refer to
  int n_cells = 0, cap_cells = 0;
  unsigned accumulate_frames = 0;
  unsigned long long* keys = nullptr;  // [cap_cells] cell key, ascending
  unsigned long long* ids = nullptr;   // [cap_cells] slot << 32 | epoch
  DevBuf cells_buf;
  // analysis (valid when analyzed)
  int analyzed = 0;
  ll_keyframe_info info = {};
  int* type = nullptr; float4* vec = nullptr; float* img = nullptr;   // img: counts line, counts plane, blurred line, blurred plane (KF_PIX each)
  float4* cloud = nullptr;             // line points, then plane points, then all points
  DevBuf res_buf;
};

// ---- append ------------------------------------------------------------------------------------------------------------------------------
__global__ void kf_count_kernel(const int* __restrict__ pt_slot, int base, int n, int* __restrict__ cnt) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const int s = pt_slot[base + t];
  if (s >= 0) atomicAdd(&cnt[s], 1);
}
__global__ void kf_flag_cells_kernel(const int* __restrict__ cnt, int cap, int thr, unsigned char* __restrict__ f) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < cap) f[s] = cnt[s] >= thr ? 1 : 0;
}
__global__ void kf_gather_cells_kernel(const int* __restrict__ slots, const int* __restrict__ d_n, const unsigned long long* __restrict__ keys, const int* __restrict__ epoch,
                                       unsigned long long* __restrict__ ok, unsigned long long* __restrict__ oid) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= *d_n) return;
  const int s = slots[r];
  ok[r] = keys[s]; oid[r] = ((unsigned long long)(unsigned)s << 32) | (unsigned)epoch[s];
}
// after a stable sort by key of (the keyframe's cells, then the new ones): a cell already held sits right before its repeat
__global__ void kf_unique_flags_kernel(const unsigned long long* __restrict__ k, const unsigned long long* __restrict__ id, int n, unsigned char* __restrict__ f) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) f[r] = (r == 0 || k[r] != k[r - 1] || id[r] != id[r - 1]) ? 1 : 0;
}
__global__ void kf_gather_pairs_kernel(const unsigned long long* __restrict__ k, const unsigned long long* __restrict__ id, const int* __restrict__ idx, int n,
                                       unsigned long long* __restrict__ ok, unsigned long long* __restrict__ oid) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) { ok[r] = k[idx[r]]; oid[r] = id[idx[r]]; }
}

// ---- analyze ------------------------------------------------------------------------------------------------------------------------------
__global__ void kf_first_of_slot_kernel(const unsigned long long* __restrict__ k, const unsigned long long* __restrict__ id, int n, int* __restrict__ first) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n && (r == 0 || k[r] != k[r - 1])) first[(int)(id[r] >> 32)] = r;
}
// the keyframe cell of every stored point (-1: none); a slot's incarnations are adjacent in the keyframe's list
__global__ void kf_point_cell_kernel(const int* __restrict__ pt_slot, const int* __restrict__ pt_epoch, int n, const int* __restrict__ first, const unsigned long long* __restrict__ k,
                                     const unsigned long long* __restrict__ id, int n_cells, int* __restrict__ cell, unsigned char* __restrict__ f) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const int s = pt_slot[t];
  int c = -1;
  if (s >= 0) {
    int r = first[s];
    if (r >= 0) {
      const unsigned long long key = k[r];
      for (; r < n_cells && k[r] == key; r++) if ((int)(unsigned)(id[r] & 0xffffffffull) == pt_epoch[t]) { c = r; break; }
    }
  }
  cell[t] = c; f[t] = c >= 0 ? 1 : 0;
}
__global__ void kf_gather_cell_of_kernel(const int* __restrict__ cell, const int* __restrict__ idx, int n, int* __restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) out[r] = cell[idx[r]];
}
__global__ void kf_segments_kernel(const int* __restrict__ c, int n, int* __restrict__ begin, int* __restrict__ end) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  if (r == 0 || c[r] != c[r - 1]) begin[c[r]] = r;
  if (r == n - 1 || c[r] != c[r + 1]) end[c[r]] = r + 1;
}

// Symmetric 3x3 eigen-decomposition in fp64 by cyclic Jacobi rotations; values ascending, vector k in column k of V, each vector's component of
// largest magnitude positive (first of equals).  The oracle runs the same arithmetic (orc_keyframe.hpp, jacobi_eig3).
__host__ __device__ inline void kf_jacobi_eig3(const double Ain[9], double w[3], double V[9]) {
  double a[3][3], v[3][3];
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { a[i][j] = Ain[i * 3 + j]; v[i][j] = i == j ? 1.0 : 0.0; }
  for (int sweep = 0; sweep < 50; sweep++) {
    if (a[0][1] == 0.0 && a[0][2] == 0.0 && a[1][2] == 0.0) break;
    for (int pq = 0; pq < 3; pq++) {
      const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
      if (a[p][q] == 0.0) continue;
      const double theta = (a[q][q] - a[p][p]) / (2.0 * a[p][q]);
      double t = 1.0 / (fabs(theta) + sqrt(theta * theta + 1.0));
      if (theta < 0.0) t = -t;
      const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
      for (int k = 0; k < 3; k++) {   // A <- A J (columns p, q)
        const double akp = a[k][p], akq = a[k][q];
        a[k][p] = c * akp - s * akq; a[k][q] = s * akp + c * akq;
      }
      for (int k = 0; k < 3; k++) {   // A <- J^T A (rows p, q)
        const double apk = a[p][k], aqk = a[q][k];
        a[p][k] = c * apk - s * aqk; a[q][k] = s * apk + c * aqk;
      }
      a[p][q] = 0.0; a[q][p] = 0.0;
      for (int k = 0; k < 3; k++) {
        const double vkp = v[k][p], vkq = v[k][q];
        v[k][p] = c * vkp - s * vkq; v[k][q] = s * vkp + c * vkq;
      }
    }
  }
  int o[3] = {0, 1, 2};
  for (int i = 0; i < 3; i++) for (int j = i + 1; j < 3; j++) if (a[o[j]][o[j]] < a[o[i]][o[i]]) { const int x = o[i]; o[i] = o[j]; o[j] = x; }
  for (int c = 0; c < 3; c++) {
    const int src = o[c];
    w[c] = a[src][src];
    int m = 0;
    for (int k = 1; k < 3; k++) if (fabs(v[k][src]) > fabs(v[m][src])) m = k;
    const double sg = v[m][src] < 0.0 ? -1.0 : 1.0;
    for (int k = 0; k < 3; k++) V[k * 3 + c] = sg * v[k][src];
  }
}

// One thread per keyframe cell: mean and covariance over its points in append order (COMP_TYPE float, as the reference), then determine_feature.
//   batch (if_update_mean_and_cov_incrementally 0): mean = xyz_sum / N, cov = (sum p p^T - N mean mean^T) / (N - 1)       (:220-233, 280-310)
//   incremental (1): append_pt's recurrence (:392-414), including its get_covmat for N <= 5 (a batch covariance at 3 and 4 points, none at 5
//   and 6) -- only for a cell's first incarnation: a cell replaced by a revisit is built without the map's flag (:747) and is batch.
__global__ void kf_cell_feature_kernel(const float4* __restrict__ pts, const int* __restrict__ sidx, const int* __restrict__ begin, const int* __restrict__ end,
                                       const unsigned long long* __restrict__ keys, const unsigned long long* __restrict__ ids, int n_cells, float box, float half,
                                       int incremental, int* __restrict__ type, float4* __restrict__ vec) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_cells) return;
  const int b = begin[c], e = end[c], n = e - b;
  const bool inc = incremental && (unsigned)(ids[c] & 0xffffffffull) == 0u;
  float mean[3] = {0.f, 0.f, 0.f}, cov[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  auto batch_cov = [&](int upto, const float m[3]) {   // :289-309 over the first `upto` points, with mean m
    for (int k = 0; k < 9; k++) cov[k] = 0.f;
    if (upto <= 2) return;
    for (int r = b; r < b + upto; r++) {
      const float4 p = pts[sidx[r]]; const float q[3] = {p.x, p.y, p.z};
      for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) cov[i * 3 + j] = cov[i * 3 + j] + q[i] * q[j];
    }
    const float fn = (float)upto, fd = (float)(upto - 1);
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { cov[i * 3 + j] -= fn * (m[i] * m[j]); cov[i * 3 + j] /= fd; }
  };
  if (inc) {
    for (int r = b; r < e; r++) {
      const float4 p = pts[sidx[r]]; const float P[3] = {p.x, p.y, p.z};
      const int N = r - b;   // points before this one
      const float ml[3] = {mean[0], mean[1], mean[2]};
      const float cl[9] = {cov[0], cov[1], cov[2], cov[3], cov[4], cov[5], cov[6], cov[7], cov[8]};
      for (int i = 0; i < 3; i++) mean[i] = ((float)N * ml[i] + P[i]) / (float)(N + 1);
      if (N > 5) {
        float d1[3], d2[3];
        for (int i = 0; i < 3; i++) { d1[i] = P[i] - ml[i]; d2[i] = ml[i] - mean[i]; }
        for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++)
          cov[i * 3 + j] = ((((float)(N - 1) * cl[i * 3 + j] + d1[i] * d1[j]) + ((float)(N + 1) * d2[i]) * d2[j]) + (2.f * d2[i]) * d1[j]) / (float)N;
      } else if (N + 1 < 5) {
        batch_cov(N + 1, mean);
      }
    }
  } else {
    float s[3] = {0.f, 0.f, 0.f};
    for (int r = b; r < e; r++) { const float4 p = pts[sidx[r]]; s[0] = s[0] + p.x; s[1] = s[1] + p.y; s[2] = s[2] + p.z; }
    for (int i = 0; i < 3; i++) mean[i] = s[i] / (float)n;
    if (n >= 5) batch_cov(n, mean);
  }
  int ty = LL_CELL_SPHERE; float4 fv = make_float4(0.f, 0.f, 0.f, 0.f);
  if (n >= 5) {
    int k, j, i; cm_unpack(keys[c], k, j, i);
    const float cx = (float)i * box + half, cy = (float)j * box + half, cz = (float)k * box + half;
    const float dx = cx - mean[0], dy = cy - mean[1], dz = cz - mean[2];
    const float dn = sqrtf(dx * dx + (dy * dy + dz * dz));
    if (!((double)dn > (double)box * 0.75)) {
      double A[9], w[3], V[9];
      for (int q = 0; q < 9; q++) A[q] = (double)cov[q];
      kf_jacobi_eig3(A, w, V);
      if (w[1] * (1.0 / 3.0) > w[0]) { ty = LL_CELL_PLANE; fv = make_float4((float)V[0], (float)V[3], (float)V[6], 0.f); }
      else if (w[2] * (1.0 / 3.0) > w[1]) { ty = LL_CELL_LINE; fv = make_float4((float)V[2], (float)V[5], (float)V[8], 0.f); }
    }
  }
  type[c] = ty; vec[c] = fv;
}

// The keyframe's centre, cell distances and image basis (one thread: the sums run in cell order), then the direction counts of every line and
// plane cell.
__device__ inline float kf_dot3(const float a[3], const float b[3]) { return a[0] * b[0] + (a[1] * b[1] + a[2] * b[2]); }   // Eigen's order
__device__ inline void kf_bin(float x, float y, float z, int& pi, int& ti) {   // feature_direction (:1073-1090)
  if (x < 0) { x = -x; y = -y; z = -z; }
  const double step = M_PI / KF_RES;
  // the float overloads atan2(float, float) / asin(float) there, pinned to the correctly rounded float of the double functions (as the oracle)
  const double phi = (double)(float)atan2((double)y, (double)x) + M_PI / 2, theta = (double)(float)asin((double)z) + M_PI / 2;
  const double fp = floor(phi / step), ft = floor(theta / step);
  pi = fp != fp ? 0 : (fp < 0 ? 0 : (fp >= KF_RES ? KF_RES - 1 : (int)fp));
  ti = ft != ft ? 0 : (ft < 0 ? 0 : (ft >= KF_RES ? KF_RES - 1 : (int)ft));
}
__global__ void __launch_bounds__(256) kf_summary_kernel(const unsigned long long* __restrict__ keys, const int* __restrict__ type, const float4* __restrict__ vec, int n_cells, float box,
                                  float half, float* __restrict__ centre, float* __restrict__ dist, float* __restrict__ img) {
  __shared__ float s_c[3];
  __shared__ float s_R[9];
  if (threadIdx.x == 0) {
    float c[3] = {0.f, 0.f, 0.f};
    double M[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};   // eigen_decompose_of_featurevector: I + sum (v v^T, float) in double, plane cells
    for (int r = 0; r < n_cells; r++) {
      int k, j, i; cm_unpack(keys[r], k, j, i);
      c[0] = c[0] + ((float)i * box + half); c[1] = c[1] + ((float)j * box + half); c[2] = c[2] + ((float)k * box + half);
      if (type[r] == LL_CELL_PLANE) {
        const float4 v = vec[r]; const float q[3] = {v.x, v.y, v.z};
        for (int a = 0; a < 3; a++) for (int b2 = 0; b2 < 3; b2++) M[a * 3 + b2] = M[a * 3 + b2] + (double)(q[a] * q[b2]);
      }
    }
    const float f = (float)(1.0 / (double)(float)n_cells);
    for (int a = 0; a < 3; a++) { s_c[a] = c[a] * f; centre[a] = s_c[a]; }
    double w[3], V[9];
    kf_jacobi_eig3(M, w, V);
    // rowwise().reverse(): columns (largest, middle, smallest) as float; column 2 = column 0 x column 1 (float)
    float R0[3] = {(float)V[2], (float)V[5], (float)V[8]}, R1[3] = {(float)V[1], (float)V[4], (float)V[7]};
    for (int a = 0; a < 3; a++) { s_R[a * 3 + 0] = R0[a]; s_R[a * 3 + 1] = R1[a]; }
    s_R[0 * 3 + 2] = R0[1] * R1[2] - R0[2] * R1[1];
    s_R[1 * 3 + 2] = R0[2] * R1[0] - R0[0] * R1[2];
    s_R[2 * 3 + 2] = R0[0] * R1[1] - R0[1] * R1[0];
  }
  __syncthreads();
  for (int r = threadIdx.x; r < n_cells; r += blockDim.x) {
    int k, j, i; cm_unpack(keys[r], k, j, i);
    const float dx = ((float)i * box + half) - s_c[0], dy = ((float)j * box + half) - s_c[1], dz = ((float)k * box + half) - s_c[2];
    dist[r] = sqrtf(dx * dx + (dy * dy + dz * dz));
    const int ty = type[r];
    if (ty == LL_CELL_LINE || ty == LL_CELL_PLANE) {
      const float4 v = vec[r]; const float q[3] = {v.x, v.y, v.z};
      const float c0[3] = {s_R[0], s_R[3], s_R[6]}, c1[3] = {s_R[1], s_R[4], s_R[7]}, c2[3] = {s_R[2], s_R[5], s_R[8]};
      int pi, ti; kf_bin(kf_dot3(c0, q), kf_dot3(c1, q), kf_dot3(c2, q), pi, ti);
      atomicAdd(&img[(ty == LL_CELL_LINE ? 0 : KF_PIX) + pi * KF_RES + ti], 1.f);   // integer counts: exact in any order
    }
  }
}
// get_ratio_range_of_cell(ratio 0.9): element ceil((u - 1) * 0.9f) of the u distinct sorted distances (std::set<float>)
__global__ void kf_roi_kernel(const float* __restrict__ sorted, int n, float* __restrict__ out) {
  int u = 0;
  for (int r = 0; r < n; r++) if (r == 0 || sorted[r] != sorted[r - 1]) u++;
  const int want = (int)ceilf((float)(u - 1) * 0.9f);
  int d = -1; float v = 0.f;
  for (int r = 0; r < n; r++) if (r == 0 || sorted[r] != sorted[r - 1]) { if (++d == want) { v = sorted[r]; break; } }
  *out = v;
}
// m_ratio_nonzero_* and apply_guassian_blur(img, 4, 4) of the count images: block 0 line, block 1 plane.  The 5-pixel wrap pad covers the 9x9
// kernel's radius, so the crop is a circular separable convolution: rows (along theta) first, then columns, float sums in tap order.
struct KfGauss { float k[9]; };
__global__ void kf_blur_kernel(float* __restrict__ img, KfGauss g, float* __restrict__ ratio) {
  __shared__ float src[KF_PIX], tmp[KF_PIX];
  __shared__ int nz;
  const float* in = img + blockIdx.x * KF_PIX; float* out = img + (2 + blockIdx.x) * KF_PIX;
  if (threadIdx.x == 0) nz = 0;
  __syncthreads();
  int my = 0;
  for (int p = threadIdx.x; p < KF_PIX; p += blockDim.x) { src[p] = in[p]; my += in[p] >= 1.f ? 1 : 0; }
  atomicAdd(&nz, my);
  __syncthreads();
  if (threadIdx.x == 0) ratio[blockIdx.x] = (float)nz / (float)KF_PIX;
  for (int p = threadIdx.x; p < KF_PIX; p += blockDim.x) {
    const int r = p / KF_RES, c = p % KF_RES;
    float s = 0.f;
    for (int t = 0; t < 9; t++) s = s + g.k[t] * src[r * KF_RES + (c + t - 4 + KF_RES) % KF_RES];
    tmp[p] = s;
  }
  __syncthreads();
  for (int p = threadIdx.x; p < KF_PIX; p += blockDim.x) {
    const int r = p / KF_RES, c = p % KF_RES;
    float s = 0.f;
    for (int t = 0; t < 9; t++) s = s + g.k[t] * tmp[((r + t - 4 + KF_RES) % KF_RES) * KF_RES + c];
    out[p] = s;
  }
}
__global__ void kf_cloud_flags_kernel(const int* __restrict__ cell_of, const int* __restrict__ type, int n, unsigned char* __restrict__ fl, unsigned char* __restrict__ fp) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const int t = type[cell_of[r]];
  fl[r] = t == LL_CELL_LINE ? 1 : 0; fp[r] = t == LL_CELL_PLANE ? 1 : 0;
}
__global__ void kf_gather_cloud_kernel(const float4* __restrict__ pts, const int* __restrict__ sidx, const int* __restrict__ sel, const int* __restrict__ d_n, int n_max,
                                       float4* __restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = d_n ? *d_n : n_max;
  if (r >= n) return;
  const float4 p = pts[sidx[sel ? sel[r] : r]];
  out[r] = make_float4(p.x, p.y, p.z, 0.f);
}

// ---- search -------------------------------------------------------------------------------------------------------------------------------
// max_similiarity_of_two_image: cv::matchTemplate(pad(img_b, 30, 30), img_a, CV_TM_CCORR_NORMED), max over the 61 x 61 positions.  One CTA per
// (earlier keyframe, image); the template and the padded image in shared memory (72 KB); one thread per position, float sums in row-major order;
// the normalisation as OpenCV's (double): num / sqrt(sum I^2 * sum T^2) when |num| < that, +-1 below 1.125 times it, else 0 (so 0 at a zero norm).
__global__ void __launch_bounds__(KF_SEARCH_THREADS) kf_search_kernel(const float* const* __restrict__ imgs, int newest, float* __restrict__ sims) {
  extern __shared__ float sm[];
  float* T = sm; float* P = sm + KF_PIX;
  __shared__ float s_tn;
  __shared__ float s_max[KF_SEARCH_THREADS / 32];
  const int his = blockIdx.x, which = blockIdx.y;   // which: 0 plane, 1 line
  const float* a = imgs[2 * newest + which];
  const float* b = imgs[2 * his + which];
  for (int p = threadIdx.x; p < KF_PIX; p += blockDim.x) T[p] = a[p];
  for (int p = threadIdx.x; p < KF_PW * KF_PW; p += blockDim.x) {
    const int r = p / KF_PW, c = p % KF_PW;
    P[p] = b[((r + KF_PAD) % KF_RES) * KF_RES + (c + KF_PAD) % KF_RES];
  }
  __syncthreads();
  if (threadIdx.x == 0) { float s = 0.f; for (int p = 0; p < KF_PIX; p++) s = s + T[p] * T[p]; s_tn = s; }
  __syncthreads();
  const double tn = (double)s_tn;
  float best = 0.f; bool any = false;
  for (int q = threadIdx.x; q < KF_POS * KF_POS; q += blockDim.x) {
    const int y = q / KF_POS, x = q % KF_POS;
    float num = 0.f, den = 0.f;
    for (int r = 0; r < KF_RES; r++) {
      const float* row = P + (y + r) * KF_PW + x; const float* tr = T + r * KF_RES;
      for (int c = 0; c < KF_RES; c++) { const float v = row[c]; num = num + tr[c] * v; den = den + v * v; }
    }
    const double t = sqrt((double)den * tn);
    double v = num;
    if (fabs(v) < t) v = v / t; else if (fabs(v) < t * 1.125) v = v > 0 ? 1.0 : -1.0; else v = 0.0;
    const float fv = (float)v;
    if (!any || fv > best) { best = fv; any = true; }
  }
  for (int o = 16; o > 0; o >>= 1) { const float w = __shfl_xor_sync(0xffffffffu, best, o); best = w > best ? w : best; }
  if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = s_max[0];
    for (int w = 1; w < KF_SEARCH_THREADS / 32; w++) m = s_max[w] > m ? s_max[w] : m;
    sims[2 * his + which] = m;
  }
}

// ---- host ---------------------------------------------------------------------------------------------------------------------------------
static KfGauss kf_gauss() {   // cv::getGaussianKernel(9, 4, CV_32F): exp(-x^2 / (2 sigma^2)) normalised in double, then float
  double t[9], s = 0.0; KfGauss g;
  for (int i = 0; i < 9; i++) { const double x = i - 4.0; t[i] = exp(-x * x / (2.0 * 16.0)); s += t[i]; }
  for (int i = 0; i < 9; i++) g.k[i] = (float)(t[i] / s);
  return g;
}
static int kf_reserve_cells(ll_ctx* ctx, ll_keyframe* kf, int need) {
  if (need <= kf->cap_cells) return LL_OK;
  int cap = kf->cap_cells > 0 ? kf->cap_cells : 4096; while (cap < need) cap *= 2;
  DevBuf nb; unsigned long long* nk = nullptr; unsigned long long* ni = nullptr;
  LL_CUDA(ctx, nb.carve([&](Carve& c) { nk = c.take<unsigned long long>(cap); ni = c.take<unsigned long long>(cap); }));
  if (kf->n_cells > 0) {
    LL_CUDA(ctx, cudaMemcpyAsync(nk, kf->keys, (size_t)kf->n_cells * 8, cudaMemcpyDeviceToDevice, ctx->stream));
    LL_CUDA(ctx, cudaMemcpyAsync(ni, kf->ids, (size_t)kf->n_cells * 8, cudaMemcpyDeviceToDevice, ctx->stream));
    LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  kf->cells_buf.release(); kf->cells_buf = nb; kf->keys = nk; kf->ids = ni; kf->cap_cells = cap;
  return LL_OK;
}

extern "C" {

int ll_keyframe_create(ll_ctx* ctx, ll_keyframe** out) {
  if (!ctx || !out) return LL_ERR_INVALID;
  ll_keyframe* kf = new ll_keyframe(); kf->device = ctx->device;
  *out = kf; return LL_OK;
}
void ll_keyframe_release(ll_keyframe* kf) {
  if (!kf) return;
  cudaSetDevice(kf->device);
  kf->cells_buf.release(); kf->res_buf.release(); delete kf;
}

int ll_keyframe_append(ll_ctx* ctx, ll_cellmap* m, const void* pts, size_t n, int fmt, int where, ll_keyframe* const* open, int n_open) {
  if (!ctx || !m || n_open < 0 || (n_open > 0 && !open)) return LL_ERR_INVALID;
  for (int k = 0; k < n_open; k++) {
    if (!open[k] || (open[k]->map && open[k]->map != m)) { ctx->set_error("keyframe is null or belongs to another cell map"); return LL_ERR_INVALID; }
    if (open[k]->map && open[k]->generation != m->generation) { ctx->set_error(KF_STALE); return LL_ERR_INVALID; }
    for (int l = 0; l < k; l++) if (open[l] == open[k]) { ctx->set_error("keyframe listed twice"); return LL_ERR_INVALID; }
  }
  cudaSetDevice(ctx->device);
  const int base = m->n_pts; const bool first = m->n_cells == 0;
  const int rc = ll_cellmap_append(ctx, m, pts, n, fmt, where);
  if (rc != LL_OK && !(rc == LL_ERR_INVALID && m->n_pts == base + (int)n)) return rc;   // out-of-range points: the append completed without them
  const std::string msg = ctx->err;
  for (int k = 0; k < n_open; k++) { open[k]->map = m; open[k]->generation = m->generation; open[k]->accumulate_frames++; open[k]->analyzed = 0; }
  if (n == 0 || n_open == 0) return rc;
  cudaStream_t s = ctx->stream;
  const int T = m->table_cap;
  int cap_c = 0; for (int k = 0; k < n_open; k++) if (open[k]->n_cells > cap_c) cap_c = open[k]->n_cells;
  const int M = cap_c + T;   // a merge holds one keyframe's cells and at most every cell of the map
  size_t cub_a = 0, cub_b = 0;
  cub::DeviceSelect::Flagged(nullptr, cub_a, cub::CountingInputIterator<int>(0), (unsigned char*)nullptr, (int*)nullptr, (int*)nullptr, M);
  cub::DeviceRadixSort::SortPairs(nullptr, cub_b, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (unsigned long long*)nullptr, M, 0, 64);
  const size_t cub_bytes = cub_a > cub_b ? cub_a : cub_b;
  int* cnt; unsigned char* f; int* sel; unsigned long long *nk, *ni, *k2, *i2, *k3, *i3; int* d_n; char* cub_tmp;
  LL_CUDA(ctx, ctx->scratch.carve([&](Carve& c) {
    cnt = c.take<int>(T); f = c.take<unsigned char>(M); sel = c.take<int>(M); nk = c.take<unsigned long long>(M); ni = c.take<unsigned long long>(M);
    k2 = c.take<unsigned long long>(M); i2 = c.take<unsigned long long>(M); k3 = c.take<unsigned long long>(M); i3 = c.take<unsigned long long>(M);
    d_n = c.take<int>(4); cub_tmp = c.take<char>(cub_bytes);
  }));
  size_t cb = cub_bytes;
  // the cells of this append: every touched cell on set_point_cloud, else those with >= 3 of its points (:656-664)
  LL_CUDA(ctx, cudaMemsetAsync(cnt, 0, (size_t)T * 4, s));
  kf_count_kernel<<<ll_div_up((int)n, 256), 256, 0, s>>>(m->pt_slot, base, (int)n, cnt);
  kf_flag_cells_kernel<<<ll_div_up(T, 256), 256, 0, s>>>(cnt, T, first ? 1 : 3, f);
  LL_CUDA(ctx, cub::DeviceSelect::Flagged(cub_tmp, cb, cub::CountingInputIterator<int>(0), f, sel, d_n, T, s));
  int h_n = 0;
  LL_CUDA(ctx, cudaMemcpyAsync(&h_n, d_n, 4, cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  ctx->launches += 3;
  if (h_n == 0) { LL_CUDA(ctx, cudaGetLastError()); return rc; }
  kf_gather_cells_kernel<<<ll_div_up(h_n, 256), 256, 0, s>>>(sel, d_n, m->keys, m->epoch, k2, i2);
  LL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(cub_tmp, cb, k2, nk, i2, ni, h_n, 0, 64, s));
  ctx->launches += 2;
  // add_cells on each open keyframe: merge into its (key, epoch)-sorted list
  for (int q = 0; q < n_open; q++) {
    ll_keyframe* kf = open[q];
    const int c0 = kf->n_cells, tot = c0 + h_n;
    if (c0 > 0) {
      LL_CUDA(ctx, cudaMemcpyAsync(k2, kf->keys, (size_t)c0 * 8, cudaMemcpyDeviceToDevice, s));
      LL_CUDA(ctx, cudaMemcpyAsync(i2, kf->ids, (size_t)c0 * 8, cudaMemcpyDeviceToDevice, s));
    }
    LL_CUDA(ctx, cudaMemcpyAsync(k2 + c0, nk, (size_t)h_n * 8, cudaMemcpyDeviceToDevice, s));
    LL_CUDA(ctx, cudaMemcpyAsync(i2 + c0, ni, (size_t)h_n * 8, cudaMemcpyDeviceToDevice, s));
    LL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(cub_tmp, cb, k2, k3, i2, i3, tot, 0, 64, s));   // stable: held cells before new ones
    kf_unique_flags_kernel<<<ll_div_up(tot, 256), 256, 0, s>>>(k3, i3, tot, f);
    LL_CUDA(ctx, cub::DeviceSelect::Flagged(cub_tmp, cb, cub::CountingInputIterator<int>(0), f, sel, d_n, tot, s));
    int u = 0;
    LL_CUDA(ctx, cudaMemcpyAsync(&u, d_n, 4, cudaMemcpyDeviceToHost, s));
    LL_CUDA(ctx, cudaStreamSynchronize(s));
    LL_TRY(kf_reserve_cells(ctx, kf, u));
    kf_gather_pairs_kernel<<<ll_div_up(u, 256), 256, 0, s>>>(k3, i3, sel, u, kf->keys, kf->ids);
    kf->n_cells = u;
    ctx->launches += 4;
  }
  LL_CUDA(ctx, cudaGetLastError());
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  if (rc != LL_OK) ctx->set_error(msg);
  return rc;
}

int ll_keyframe_analyze(ll_ctx* ctx, ll_cellmap* m, ll_keyframe* kf, int incremental_cov, ll_keyframe_info* info) {
  if (!ctx || !m || !kf || (kf->map && kf->map != m)) return LL_ERR_INVALID;
  if (kf->map && kf->generation != m->generation) { ctx->set_error(KF_STALE); return LL_ERR_INVALID; }
  cudaSetDevice(ctx->device);
  cudaStream_t s = ctx->stream;
  const int C = kf->n_cells, N = m->n_pts, T = m->table_cap;
  ll_keyframe_info in = {};
  in.cells = C; in.accumulate_frames = (int)kf->accumulate_frames;
  if (C == 0) { kf->info = in; kf->analyzed = 1; kf->type = nullptr; if (info) *info = in; return LL_OK; }   // no cell: nothing to type (roi 0)
  const float box = m->resolution * 1.0f, half = m->resolution * 0.5f;
  size_t cub_a = 0, cub_b = 0, cub_c = 0;
  const int big = N > C ? N : C;
  cub::DeviceSelect::Flagged(nullptr, cub_a, cub::CountingInputIterator<int>(0), (unsigned char*)nullptr, (int*)nullptr, (int*)nullptr, big);
  cub::DeviceRadixSort::SortPairs(nullptr, cub_b, (int*)nullptr, (int*)nullptr, (int*)nullptr, (int*)nullptr, N, 0, 32);
  cub::DeviceRadixSort::SortKeys(nullptr, cub_c, (float*)nullptr, (float*)nullptr, C);
  size_t cub_bytes = cub_a > cub_b ? cub_a : cub_b; if (cub_c > cub_bytes) cub_bytes = cub_c;
  int *first, *cell, *sel, *cell_of, *cell_of2, *sidx, *begin, *end, *d_n; unsigned char *f, *f2; float *vals, *dist, *dist_sorted; char* cub_tmp;
  LL_CUDA(ctx, ctx->scratch.carve([&](Carve& c) {
    first = c.take<int>(T); cell = c.take<int>(N); f = c.take<unsigned char>(big); f2 = c.take<unsigned char>(N); sel = c.take<int>(big); cell_of = c.take<int>(N);
    cell_of2 = c.take<int>(N); sidx = c.take<int>(N); begin = c.take<int>(C); end = c.take<int>(C); vals = c.take<float>(8); dist = c.take<float>(C); dist_sorted = c.take<float>(C);
    d_n = c.take<int>(4); cub_tmp = c.take<char>(cub_bytes);
  }));
  size_t cb = cub_bytes;
  // 1. the keyframe cell of every stored point; the keyframe's points sorted by (cell, store order)
  LL_CUDA(ctx, cudaMemsetAsync(first, 0xff, (size_t)T * 4, s));
  kf_first_of_slot_kernel<<<ll_div_up(C, 256), 256, 0, s>>>(kf->keys, kf->ids, C, first);
  kf_point_cell_kernel<<<ll_div_up(N, 256), 256, 0, s>>>(m->pt_slot, m->pt_epoch, N, first, kf->keys, kf->ids, C, cell, f);
  LL_CUDA(ctx, cub::DeviceSelect::Flagged(cub_tmp, cb, cub::CountingInputIterator<int>(0), f, sel, d_n, N, s));
  int n_sel = 0;
  LL_CUDA(ctx, cudaMemcpyAsync(&n_sel, d_n, 4, cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  ctx->launches += 3;
  kf_gather_cell_of_kernel<<<ll_div_up(n_sel, 256), 256, 0, s>>>(cell, sel, n_sel, cell_of);
  int bits = 1; while ((1 << bits) < C) bits++;
  LL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(cub_tmp, cb, cell_of, cell_of2, sel, sidx, n_sel, 0, bits, s));
  LL_CUDA(ctx, cudaMemsetAsync(begin, 0, (size_t)C * 4, s));
  LL_CUDA(ctx, cudaMemsetAsync(end, 0, (size_t)C * 4, s));
  kf_segments_kernel<<<ll_div_up(n_sel, 256), 256, 0, s>>>(cell_of2, n_sel, begin, end);
  // results: types, vectors, 4 images, the three clouds
  float4* cloud = nullptr;
  LL_CUDA(ctx, kf->res_buf.carve([&](Carve& c) {
    kf->type = c.take<int>(C); kf->vec = c.take<float4>(C); kf->img = c.take<float>(4 * KF_PIX); cloud = c.take<float4>(2 * (size_t)n_sel);
  }));
  // 2. per cell: mean, covariance, type
  kf_cell_feature_kernel<<<ll_div_up(C, 128), 128, 0, s>>>(m->pts, sidx, begin, end, kf->keys, kf->ids, C, box, half, incremental_cov ? 1 : 0, kf->type, kf->vec);
  // 3. centre, distances, direction counts; ROI range; ratios and blur.  vals: centre xyz, roi range, ratio line, ratio plane
  LL_CUDA(ctx, cudaMemsetAsync(kf->img, 0, 2 * KF_PIX * 4, s));
  kf_summary_kernel<<<1, 256, 0, s>>>(kf->keys, kf->type, kf->vec, C, box, half, vals, dist, kf->img);
  LL_CUDA(ctx, cub::DeviceRadixSort::SortKeys(cub_tmp, cb, dist, dist_sorted, C, 0, 32, s));
  kf_roi_kernel<<<1, 1, 0, s>>>(dist_sorted, C, vals + 3);
  kf_blur_kernel<<<2, 512, 0, s>>>(kf->img, kf_gauss(), vals + 4);
  // 4. typed clouds: line, plane (cell order, append order inside a cell), all
  kf_cloud_flags_kernel<<<ll_div_up(n_sel, 256), 256, 0, s>>>(cell_of2, kf->type, n_sel, f, f2);
  LL_CUDA(ctx, cub::DeviceSelect::Flagged(cub_tmp, cb, cub::CountingInputIterator<int>(0), f, sel, d_n, n_sel, s));
  kf_gather_cloud_kernel<<<ll_div_up(n_sel, 256), 256, 0, s>>>(m->pts, sidx, sel, d_n, n_sel, cloud);
  int h[2] = {0, 0};
  LL_CUDA(ctx, cudaMemcpyAsync(h, d_n, 4, cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  LL_CUDA(ctx, cub::DeviceSelect::Flagged(cub_tmp, cb, cub::CountingInputIterator<int>(0), f2, sel, d_n + 1, n_sel, s));
  kf_gather_cloud_kernel<<<ll_div_up(n_sel, 256), 256, 0, s>>>(m->pts, sidx, sel, d_n + 1, n_sel, cloud + h[0]);
  LL_CUDA(ctx, cudaMemcpyAsync(h + 1, d_n + 1, 4, cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  kf_gather_cloud_kernel<<<ll_div_up(n_sel, 256), 256, 0, s>>>(m->pts, sidx, nullptr, nullptr, n_sel, cloud + h[0] + h[1]);
  ctx->launches += 14;
  kf->cloud = cloud;
  float hv[6];
  std::vector<int> ht(C);
  LL_CUDA(ctx, cudaMemcpyAsync(hv, vals, sizeof(hv), cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaMemcpyAsync(ht.data(), kf->type, (size_t)C * 4, cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaGetLastError());
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  for (int a = 0; a < 3; a++) in.center[a] = hv[a];
  in.roi_range = hv[3]; in.ratio_nonzero_line = hv[4]; in.ratio_nonzero_plane = hv[5];
  for (int v : ht) { in.line_cells += v == LL_CELL_LINE; in.plane_cells += v == LL_CELL_PLANE; }
  in.line_points = (size_t)h[0]; in.plane_points = (size_t)h[1]; in.all_points = (size_t)n_sel;
  kf->info = in; kf->analyzed = 1;
  if (info) *info = in;
  return LL_OK;
}

int ll_keyframe_get_info(const ll_keyframe* kf, ll_keyframe_info* info) {
  if (!kf || !info || !kf->analyzed) return LL_ERR_INVALID;
  *info = kf->info;
  return LL_OK;
}

int ll_keyframe_cells(ll_ctx* ctx, const ll_keyframe* kf, uint64_t* keys, int* epochs, int* types, float* vecs, int cap, int* n) {
  if (!ctx || !kf || !n || cap < 0) return LL_ERR_INVALID;
  *n = kf->n_cells;
  const int w = kf->n_cells < cap ? kf->n_cells : cap;
  if (w == 0) return LL_OK;
  if ((types || vecs) && !kf->analyzed) { ctx->set_error("keyframe not analyzed since its last append"); return LL_ERR_INVALID; }
  cudaSetDevice(ctx->device);
  std::vector<unsigned long long> ids(w);
  std::vector<float4> v(vecs ? w : 0);
  if (keys) LL_CUDA(ctx, cudaMemcpyAsync(keys, kf->keys, (size_t)w * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (epochs) LL_CUDA(ctx, cudaMemcpyAsync(ids.data(), kf->ids, (size_t)w * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (types) LL_CUDA(ctx, cudaMemcpyAsync(types, kf->type, (size_t)w * 4, cudaMemcpyDeviceToHost, ctx->stream));
  if (vecs) LL_CUDA(ctx, cudaMemcpyAsync(v.data(), kf->vec, (size_t)w * 16, cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (epochs) for (int r = 0; r < w; r++) epochs[r] = (int)(unsigned)(ids[r] & 0xffffffffull);
  if (vecs) for (int r = 0; r < w; r++) { vecs[3 * r] = v[r].x; vecs[3 * r + 1] = v[r].y; vecs[3 * r + 2] = v[r].z; }
  return LL_OK;
}

int ll_keyframe_images(ll_ctx* ctx, const ll_keyframe* kf, float* count_line, float* count_plane, float* line, float* plane) {
  if (!ctx || !kf) return LL_ERR_INVALID;
  if (!kf->analyzed) { ctx->set_error("keyframe not analyzed since its last append"); return LL_ERR_INVALID; }
  float* dst[4] = {count_line, count_plane, line, plane};
  for (int k = 0; k < 4; k++) {
    if (!dst[k]) continue;
    if (kf->n_cells == 0) memset(dst[k], 0, KF_PIX * 4);
    else LL_CUDA(ctx, cudaMemcpyAsync(dst[k], kf->img + k * KF_PIX, KF_PIX * 4, cudaMemcpyDeviceToHost, ctx->stream));
  }
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return LL_OK;
}

int ll_keyframe_cloud(ll_ctx* ctx, const ll_keyframe* kf, int which, ll_point* out_host, size_t cap, size_t* n_out, const ll_point** out_dev) {
  if (!ctx || !kf || !n_out || !(which == LL_CELL_LINE || which == LL_CELL_PLANE || which == LL_CELL_ALL)) return LL_ERR_INVALID;
  if (!kf->analyzed) { ctx->set_error("keyframe not analyzed since its last append"); return LL_ERR_INVALID; }
  const ll_keyframe_info& in = kf->info;
  const size_t off = which == LL_CELL_LINE ? 0 : (which == LL_CELL_PLANE ? in.line_points : in.line_points + in.plane_points);
  const size_t n = which == LL_CELL_LINE ? in.line_points : (which == LL_CELL_PLANE ? in.plane_points : in.all_points);
  *n_out = n;
  const ll_point* d = n ? (const ll_point*)(kf->cloud + off) : nullptr;
  if (out_dev) *out_dev = d;
  if (out_host && n) {
    LL_CUDA(ctx, cudaMemcpyAsync(out_host, d, (n < cap ? n : cap) * 16, cudaMemcpyDeviceToHost, ctx->stream));
    LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  return LL_OK;
}

void ll_loop_cfg_default(ll_loop_cfg* c) {
  c->minimum_keyframe_differen = 200;    // loop_closure/minimum_keyframe_differen (rosbag_loop.launch, both YAMLs)
  c->avail_ratio_plane = 0.05f;          // laser_mapping.hpp:894
  c->avail_ratio_line = 0.03f;           // :895
  c->maximum_roi_difference = 5.0f;      // :1004
  c->minimum_similarity_linear = 0.65f;  // loop_closure/minimum_similarity_linear (YAMLs)
  c->minimum_similarity_planar = 0.94f;  // loop_closure/minimum_similarity_planar (YAMLs)
  c->plane_with_line = 0.92;             // :1012
}

int ll_loop_search(ll_ctx* ctx, const ll_keyframe* const* kfs, int n, int newest, const ll_loop_cfg* cfg, float* sim_plane, float* sim_line, int* candidates,
                   int* n_candidates) {
  if (!ctx || !kfs || !cfg || !n_candidates || newest < 0 || newest >= n) return LL_ERR_INVALID;
  for (int k = 0; k <= newest; k++)
    if (!kfs[k] || !kfs[k]->analyzed) { ctx->set_error("keyframe missing or not analyzed since its last append"); return LL_ERR_INVALID; }
  *n_candidates = 0;
  if (newest == 0) return LL_OK;
  cudaSetDevice(ctx->device);
  cudaStream_t s = ctx->stream;
  const size_t smem = (size_t)(KF_PIX + KF_PW * KF_PW) * 4;
  LL_CUDA(ctx, cudaFuncSetAttribute(kf_search_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // image table: plane, line of every keyframe up to `newest` (a keyframe without cells has all-zero images)
  const float** tab = nullptr; float* sims = nullptr; float* zero = nullptr;
  LL_CUDA(ctx, ctx->scratch.carve([&](Carve& c) { tab = c.take<const float*>(2 * (size_t)(newest + 1)); sims = c.take<float>(2 * (size_t)newest); zero = c.take<float>(KF_PIX); }));
  std::vector<const float*> h_tab(2 * (size_t)(newest + 1));
  for (int k = 0; k <= newest; k++) {
    h_tab[2 * k] = kfs[k]->n_cells ? kfs[k]->img + 3 * KF_PIX : zero;
    h_tab[2 * k + 1] = kfs[k]->n_cells ? kfs[k]->img + 2 * KF_PIX : zero;
  }
  LL_CUDA(ctx, cudaMemsetAsync(zero, 0, KF_PIX * 4, s));
  LL_CUDA(ctx, cudaMemcpyAsync(tab, h_tab.data(), h_tab.size() * sizeof(float*), cudaMemcpyHostToDevice, s));
  kf_search_kernel<<<dim3(newest, 2), KF_SEARCH_THREADS, smem, s>>>(tab, newest, sims);
  ctx->launches++;
  std::vector<float> h(2 * (size_t)newest);
  LL_CUDA(ctx, cudaMemcpyAsync(h.data(), sims, h.size() * 4, cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaGetLastError());
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  // the gates of :994-1033, his ascending
  const ll_keyframe_info& last = kfs[newest]->info;
  const size_t n_kf = (size_t)newest + 1;
  int nc = 0;
  for (int his = 0; his < newest; his++) {
    const float sp = h[2 * his], sl = h[2 * his + 1];
    if (sim_plane) sim_plane[his] = sp;
    if (sim_line) sim_line[his] = sl;
    const ll_keyframe_info& o = kfs[his]->info;
    if (n_kf - (size_t)his < (size_t)cfg->minimum_keyframe_differen) continue;
    if (o.ratio_nonzero_plane < cfg->avail_ratio_plane && o.ratio_nonzero_line < cfg->avail_ratio_line) continue;
    if ((double)fabsf(o.roi_range - last.roi_range) > (double)cfg->maximum_roi_difference) continue;   // abs(float) is std::abs(float) there
    if (!((sl > cfg->minimum_similarity_linear && (double)sp > cfg->plane_with_line) || sp > cfg->minimum_similarity_planar)) continue;
    // (a - b) / (a + b) * 0.1 in size_t (:1030): nonzero, so skipped, unless b <= a and b > 0 (a + b == 0 would divide by zero: skipped)
    const size_t a = (size_t)last.cells, b = (size_t)o.cells;
    if (a + b == 0 || (a - b) / (a + b)) continue;
    if (candidates) candidates[nc] = his;
    nc++;
  }
  *n_candidates = nc;
  return LL_OK;
}

}  // extern "C"

// ---- loop image (ll_mapper_loop_save / ll_mapper_loop_load, loop.cu) ---------------------------------------------------------------------
int kf_cell_count(const ll_keyframe* kf) { return kf->n_cells; }
unsigned kf_accumulate_frames(const ll_keyframe* kf) { return kf->accumulate_frames; }

int kf_cell_ids(ll_ctx* ctx, const ll_keyframe* kf, unsigned long long* keys, unsigned long long* ids) {
  if (kf->n_cells == 0) return LL_OK;
  LL_CUDA(ctx, cudaMemcpyAsync(keys, kf->keys, (size_t)kf->n_cells * 8, cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaMemcpyAsync(ids, kf->ids, (size_t)kf->n_cells * 8, cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return LL_OK;
}

int kf_restore_open(ll_ctx* ctx, ll_cellmap* m, ll_keyframe* kf, const unsigned long long* keys, const unsigned long long* ids, int n, unsigned accumulate_frames) {
  LL_TRY(kf_reserve_cells(ctx, kf, n));
  if (n > 0) {
    LL_CUDA(ctx, cudaMemcpyAsync(kf->keys, keys, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
    LL_CUDA(ctx, cudaMemcpyAsync(kf->ids, ids, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
    LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  kf->n_cells = n; kf->accumulate_frames = accumulate_frames; kf->analyzed = 0;
  kf->map = accumulate_frames > 0 ? m : nullptr;   // an append, also of no cell, binds a keyframe to its map
  kf->generation = m->generation;
  return LL_OK;
}

int kf_restore_closed(ll_ctx* ctx, ll_cellmap* m, ll_keyframe* kf, const ll_keyframe_info& info, const float* img, const void* cloud) {
  kf->map = m; kf->generation = m->generation; kf->n_cells = info.cells; kf->accumulate_frames = (unsigned)info.accumulate_frames;
  kf->info = info; kf->analyzed = 1; kf->type = nullptr; kf->vec = nullptr; kf->img = nullptr; kf->cloud = nullptr;
  if (info.cells == 0) return LL_OK;
  const size_t np = info.line_points + info.plane_points;
  float* im = nullptr; float4* cl = nullptr;
  LL_CUDA(ctx, kf->res_buf.carve([&](Carve& c) { im = c.take<float>(4 * KF_PIX); cl = c.take<float4>(np); }));
  LL_CUDA(ctx, cudaMemcpyAsync(im, img, 4 * KF_PIX * 4, cudaMemcpyHostToDevice, ctx->stream));
  if (np) LL_CUDA(ctx, cudaMemcpyAsync(cl, cloud, np * 16, cudaMemcpyHostToDevice, ctx->stream));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  kf->img = im; kf->cloud = cl;
  return LL_OK;
}
