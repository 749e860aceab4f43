// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header). PARITY UNPINNED.
// CPU restatement of the two PCL primitives on the hot path. PCL is a third-party dependency of the
// reference that is neither vendored nor version-pinned (CMakeLists.txt:25, README.md:51 recommends >= 1.9)
// and is not installed here; the published algorithms are restated.
//
//  * pcl::VoxelGrid<PointXYZI>::applyFilter (PCL 1.8+/1.9, downsample_all_data = true):
//      call sites  loam_livox/source/laser_feature_extractor.hpp:372-380,
//                  loam_livox/source/laser_mapping.hpp:491,509,533-537,1367-1373,1434-1437
//  * pcl::KdTreeFLANN<PointXYZI>::setInputCloud / nearestKSearch (FLANN KDTreeSingleIndex, L2_Simple<float>,
//    leaf_max_size 15, eps 0, sorted):
//      call sites  loam_livox/source/point_cloud_registration.hpp:249,351,596-597,
//                  loam_livox/source/laser_mapping.hpp:544-545
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <limits>
#include <numeric>
#include <vector>

namespace orc {

// ------------------------------------------------------------------ VoxelGrid
// in/out: n x 4 floats (x,y,z,intensity). Returns number of output points; `out` must hold n*4 floats.
// Within a voxel PCL sums in the (unstable) std::sort order; the oracle fixes that order to ascending
// input index (a stable sort) — the CUDA path uses the same order, so the comparison is bit-exact.
inline int voxel_grid(const float* in, int n, float leaf, float* out) {
  if (n == 0) return 0;
  const float inv = 1.0f / leaf;  // inverse_leaf_size_ = Array4f::Ones() / leaf_size_
  float mn[3] = {std::numeric_limits<float>::max(), std::numeric_limits<float>::max(), std::numeric_limits<float>::max()};
  float mx[3] = {-std::numeric_limits<float>::max(), -std::numeric_limits<float>::max(), -std::numeric_limits<float>::max()};
  int nfinite = 0;
  for (int i = 0; i < n; i++) {
    const float* p = in + (size_t)i * 4;
    if (!std::isfinite(p[0]) || !std::isfinite(p[1]) || !std::isfinite(p[2])) continue;
    nfinite++;
    for (int k = 0; k < 3; k++) { mn[k] = std::min(mn[k], p[k]); mx[k] = std::max(mx[k], p[k]); }
  }
  if (nfinite == 0) return 0;
  int64_t dx = (int64_t)((mx[0] - mn[0]) * inv) + 1, dy = (int64_t)((mx[1] - mn[1]) * inv) + 1, dz = (int64_t)((mx[2] - mn[2]) * inv) + 1;
  if (dx * dy * dz > (int64_t)std::numeric_limits<int32_t>::max()) {  // PCL: warn and pass the input through
    std::copy(in, in + (size_t)n * 4, out);
    return n;
  }
  int min_b[3], max_b[3], div_b[3];
  for (int k = 0; k < 3; k++) { min_b[k] = (int)std::floor(mn[k] * inv); max_b[k] = (int)std::floor(mx[k] * inv); div_b[k] = max_b[k] - min_b[k] + 1; }
  const int mul[3] = {1, div_b[0], div_b[0] * div_b[1]};
  std::vector<std::pair<unsigned, int>> iv; iv.reserve(n);
  for (int i = 0; i < n; i++) {
    const float* p = in + (size_t)i * 4;
    if (!std::isfinite(p[0]) || !std::isfinite(p[1]) || !std::isfinite(p[2])) continue;
    int ijk0 = (int)(std::floor(p[0] * inv) - (float)min_b[0]);
    int ijk1 = (int)(std::floor(p[1] * inv) - (float)min_b[1]);
    int ijk2 = (int)(std::floor(p[2] * inv) - (float)min_b[2]);
    iv.emplace_back((unsigned)(ijk0 * mul[0] + ijk1 * mul[1] + ijk2 * mul[2]), i);
  }
  std::stable_sort(iv.begin(), iv.end(), [](const std::pair<unsigned, int>& a, const std::pair<unsigned, int>& b) { return a.first < b.first; });
  int m = 0; size_t index = 0;
  while (index < iv.size()) {
    size_t i = index + 1;
    while (i < iv.size() && iv[i].first == iv[index].first) ++i;
    // CentroidPoint<PointXYZI>: AccumulatorXYZ (Vector3f sum) + AccumulatorIntensity (float sum), divided by n
    float s[4] = {0.f, 0.f, 0.f, 0.f};
    for (size_t li = index; li < i; li++) { const float* p = in + (size_t)iv[li].second * 4; s[0] += p[0]; s[1] += p[1]; s[2] += p[2]; s[3] += p[3]; }
    const float cnt = (float)(i - index);
    out[(size_t)m * 4 + 0] = s[0] / cnt; out[(size_t)m * 4 + 1] = s[1] / cnt; out[(size_t)m * 4 + 2] = s[2] / cnt; out[(size_t)m * 4 + 3] = s[3] / cnt;
    m++; index = i;
  }
  return m;
}

// ------------------------------------------------------------------ exact k-NN
// FLANN L2_Simple<float>: result += diff*diff over x,y,z, float accumulation, no FMA (built -ffp-contract=off).
inline float dist2(const float* a, const float* b) {
  float r = 0.f; float d = a[0] - b[0]; r += d * d; d = a[1] - b[1]; r += d * d; d = a[2] - b[2]; r += d * d; return r;
}

// k best (d2, idx) kept sorted ascending, ties broken by smaller index (FLANN leaves ties unspecified).
struct KnnHeap {
  int k, cnt; float* d; int* id;
  KnnHeap(int k_, float* d_, int* id_) : k(k_), cnt(0), d(d_), id(id_) {}
  inline float worst() const { return cnt < k ? std::numeric_limits<float>::infinity() : d[k - 1]; }
  inline void push(float dd, int ii) {
    if (cnt == k) { if (!(dd < d[k - 1] || (dd == d[k - 1] && ii < id[k - 1]))) return; }
    else cnt++;
    int j = cnt - 1;
    while (j > 0 && (d[j - 1] > dd || (d[j - 1] == dd && id[j - 1] > ii))) { d[j] = d[j - 1]; id[j] = id[j - 1]; j--; }
    d[j] = dd; id[j] = ii;
  }
};

// Bucketed KD-tree (leaf <= 15 points as PCL passes to FLANN), split at the median of the widest dimension.
// Tree shape differs from FLANN's middleSplit but the search is exact (eps = 0), so results are identical up to ties.
struct KdTree {
  struct Node { int left, right; int dim; float split_lo, split_hi; int begin, end; };
  std::vector<float> pts;  // reordered copy, n x 3
  std::vector<int> ids;    // original index of reordered point
  std::vector<Node> nodes; int n = 0; float bb_lo[3], bb_hi[3];
  static constexpr int kLeaf = 15;

  void build(const float* p4, int n_) {  // p4: n x 4 (x,y,z,intensity); non-finite points are skipped like PCL
    std::vector<int> idx; idx.reserve(n_);
    for (int i = 0; i < n_; i++) { const float* p = p4 + (size_t)i * 4; if (std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2])) idx.push_back(i); }
    n = (int)idx.size(); nodes.clear(); nodes.reserve(2 * (n / kLeaf + 2));
    for (int k = 0; k < 3; k++) { bb_lo[k] = std::numeric_limits<float>::max(); bb_hi[k] = -std::numeric_limits<float>::max(); }
    for (int i : idx) for (int k = 0; k < 3; k++) { bb_lo[k] = std::min(bb_lo[k], p4[(size_t)i * 4 + k]); bb_hi[k] = std::max(bb_hi[k], p4[(size_t)i * 4 + k]); }
    if (n > 0) build_rec(p4, idx, 0, n);
    pts.resize((size_t)n * 3); ids = idx;
    for (int i = 0; i < n; i++) for (int k = 0; k < 3; k++) pts[(size_t)i * 3 + k] = p4[(size_t)idx[i] * 4 + k];
  }
  int build_rec(const float* p4, std::vector<int>& idx, int b, int e) {
    int me = (int)nodes.size(); nodes.push_back(Node());
    if (e - b <= kLeaf) { nodes[me] = {-1, -1, 0, 0.f, 0.f, b, e}; return me; }
    float lo[3], hi[3];
    for (int k = 0; k < 3; k++) { lo[k] = std::numeric_limits<float>::max(); hi[k] = -std::numeric_limits<float>::max(); }
    for (int i = b; i < e; i++) for (int k = 0; k < 3; k++) { float v = p4[(size_t)idx[i] * 4 + k]; lo[k] = std::min(lo[k], v); hi[k] = std::max(hi[k], v); }
    int dim = 0; if (hi[1] - lo[1] > hi[dim] - lo[dim]) dim = 1; if (hi[2] - lo[2] > hi[dim] - lo[dim]) dim = 2;
    int mid = (b + e) / 2;
    std::nth_element(idx.begin() + b, idx.begin() + mid, idx.begin() + e, [&](int a, int c) { return p4[(size_t)a * 4 + dim] < p4[(size_t)c * 4 + dim]; });
    float split_lo = -std::numeric_limits<float>::max(), split_hi = p4[(size_t)idx[mid] * 4 + dim];
    for (int i = b; i < mid; i++) split_lo = std::max(split_lo, p4[(size_t)idx[i] * 4 + dim]);
    int l = build_rec(p4, idx, b, mid); int r = build_rec(p4, idx, mid, e);
    nodes[me] = {l, r, dim, split_lo, split_hi, b, e};
    return me;
  }
  // Exact search. `dists` holds the per-dimension squared offsets to the current cell (as in FLANN/nanoflann).
  void search_rec(int ni, const float* q, float mindist, float* dists, KnnHeap& h) const {
    const Node& nd = nodes[ni];
    if (nd.left < 0) {
      for (int i = nd.begin; i < nd.end; i++) h.push(dist2(q, &pts[(size_t)i * 3]), ids[i]);
      return;
    }
    const float v = q[nd.dim]; const float d1 = v - nd.split_lo, d2 = v - nd.split_hi;
    int best, other; float cut;
    if (d1 + d2 < 0) { best = nd.left; other = nd.right; cut = d2 * d2; }
    else { best = nd.right; other = nd.left; cut = d1 * d1; }
    search_rec(best, q, mindist, dists, h);
    const float saved = dists[nd.dim];
    const float nm = mindist + cut - saved;
    dists[nd.dim] = cut;
    // the bound is summed in a different order than dist2(); keep a 1e-5 relative guard band so float
    // rounding can never prune a true neighbour (the result then equals brute force bit for bit)
    if (nm * 0.99999f <= h.worst()) search_rec(other, q, nm, dists, h);
    dists[nd.dim] = saved;
  }
  // returns number found (<= k); out_d / out_id sorted ascending
  int knn(const float* q, int k, int* out_id, float* out_d) const {
    KnnHeap h(k, out_d, out_id);
    if (n == 0) return 0;
    float dists[3] = {0, 0, 0}; float mind = 0;
    for (int kx = 0; kx < 3; kx++) {
      if (q[kx] < bb_lo[kx]) { dists[kx] = (q[kx] - bb_lo[kx]) * (q[kx] - bb_lo[kx]); mind += dists[kx]; }
      if (q[kx] > bb_hi[kx]) { dists[kx] = (q[kx] - bb_hi[kx]) * (q[kx] - bb_hi[kx]); mind += dists[kx]; }
    }
    search_rec(0, q, mind, dists, h);
    return h.cnt;
  }
};

inline int knn_brute(const float* map4, int n, const float* q, int k, int* out_id, float* out_d) {
  KnnHeap h(k, out_d, out_id);
  for (int i = 0; i < n; i++) {
    const float* p = map4 + (size_t)i * 4;
    if (!std::isfinite(p[0]) || !std::isfinite(p[1]) || !std::isfinite(p[2])) continue;
    h.push(dist2(q, p), i);
  }
  return h.cnt;
}

}  // namespace orc
