// ORACLE — keyframes over the full-resolution cell map, their feature images and the loop candidate search, restated from
// loam_livox/source/cell_map_keyframe.hpp (Points_cloud_cell :54-474, Points_cloud_map::append_cloud / find_cell :585-758, Maps_keyframe
// :1002-1567) and laser_mapping.hpp:988-1033, with the OpenCV calls they make (GaussianBlur, matchTemplate CCORR_NORMED) restated from
// OpenCV's published behaviour.  Pinned choices (DESIGN.md §5): cells ordered by (key, incarnation) instead of pointer order; eigenvectors
// with their largest-magnitude component positive; the cell eigen-decomposition in fp64 (cyclic Jacobi) on the float covariance; a non-finite
// point is dropped; an empty keyframe has ROI range 0.
#pragma once
#include <array>
#include <cmath>
#include <cstdint>
#include <map>
#include <memory>
#include <set>
#include <utility>
#include <vector>

namespace orc_kf {

enum { SPHERE = 0, LINE = 1, PLANE = 2 };
static const int RES = 60, PIX = RES * RES;

// Symmetric 3x3 eigen-decomposition, fp64 cyclic Jacobi: values ascending, vector c in column c of V (row-major), each vector's
// largest-magnitude component positive (first of equals).
inline void jacobi_eig3(const double Ain[9], double w[3], double V[9]) {
  double a[3][3], v[3][3];
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { a[i][j] = Ain[i * 3 + j]; v[i][j] = i == j ? 1.0 : 0.0; }
  for (int sweep = 0; sweep < 50; sweep++) {
    if (a[0][1] == 0.0 && a[0][2] == 0.0 && a[1][2] == 0.0) break;
    for (int pq = 0; pq < 3; pq++) {
      const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
      if (a[p][q] == 0.0) continue;
      const double theta = (a[q][q] - a[p][p]) / (2.0 * a[p][q]);
      double t = 1.0 / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
      if (theta < 0.0) t = -t;
      const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
      for (int k = 0; k < 3; k++) { const double akp = a[k][p], akq = a[k][q]; a[k][p] = c * akp - s * akq; a[k][q] = s * akp + c * akq; }
      for (int k = 0; k < 3; k++) { const double apk = a[p][k], aqk = a[q][k]; a[p][k] = c * apk - s * aqk; a[q][k] = s * apk + c * aqk; }
      a[p][q] = 0.0; a[q][p] = 0.0;
      for (int k = 0; k < 3; k++) { const double vkp = v[k][p], vkq = v[k][q]; v[k][p] = c * vkp - s * vkq; v[k][q] = s * vkp + c * vkq; }
    }
  }
  int o[3] = {0, 1, 2};
  for (int i = 0; i < 3; i++) for (int j = i + 1; j < 3; j++) if (a[o[j]][o[j]] < a[o[i]][o[i]]) std::swap(o[i], o[j]);
  for (int c = 0; c < 3; c++) {
    const int src = o[c];
    w[c] = a[src][src];
    int m = 0;
    for (int k = 1; k < 3; k++) if (std::fabs(v[k][src]) > std::fabs(v[m][src])) m = k;
    const double sg = v[m][src] < 0.0 ? -1.0 : 1.0;
    for (int k = 0; k < 3; k++) V[k * 3 + c] = sg * v[k][src];
  }
}

// Points_cloud_cell<float> with COMP_TYPE float, IF_COV_INIT_IDENTITY 0
struct Cell {
  uint64_t key = 0; int inc = 0;
  float center[3] = {0, 0, 0}; float res = 0.5f;
  bool incremental = false;
  std::vector<std::array<float, 3>> pts;
  float xyz_sum[3] = {0, 0, 0}, mean[3] = {0, 0, 0}, cov[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  int type = SPHERE; float vec[3] = {0, 0, 0};

  void batch_cov(size_t n) {   // get_covmat :289-309 with the current mean
    for (float& c : cov) c = 0.f;
    if (n <= 2) return;
    for (size_t r = 0; r < n; r++) for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) cov[i * 3 + j] = cov[i * 3 + j] + pts[r][i] * pts[r][j];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { cov[i * 3 + j] -= (float)n * (mean[i] * mean[j]); cov[i * 3 + j] /= (float)(n - 1); }
  }
  void append_pt(const std::array<float, 3>& P) {   // :378-419
    pts.push_back(P);
    for (int i = 0; i < 3; i++) xyz_sum[i] = xyz_sum[i] + P[i];
    if (incremental) {
      const float ml[3] = {mean[0], mean[1], mean[2]};
      float cl[9]; for (int k = 0; k < 9; k++) cl[k] = cov[k];
      const size_t N = pts.size() - 1;
      for (int i = 0; i < 3; i++) mean[i] = ((float)N * ml[i] + P[i]) / (float)(N + 1);
      if (N > 5) {
        float d1[3], d2[3];
        for (int i = 0; i < 3; i++) { d1[i] = P[i] - ml[i]; d2[i] = ml[i] - mean[i]; }
        for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++)
          cov[i * 3 + j] = ((((float)(N - 1) * cl[i * 3 + j] + d1[i] * d1[j]) + ((float)(N + 1) * d2[i]) * d2[j]) + (2.f * d2[i]) * d1[j]) / (float)N;
      } else if (pts.size() < 5) {   // get_covmat(): recomputed below 5 points only (then incremental)
        batch_cov(pts.size());
      }
    }
  }
  int determine_feature() {   // :436-473
    type = SPHERE; vec[0] = vec[1] = vec[2] = 0.f;
    if (pts.size() < 5) return type;
    if (!incremental) {   // get_mean + get_covmat
      for (int i = 0; i < 3; i++) mean[i] = xyz_sum[i] / (float)pts.size();
      batch_cov(pts.size());
    }
    const float dx = center[0] - mean[0], dy = center[1] - mean[1], dz = center[2] - mean[2];
    const float dn = std::sqrt(dx * dx + (dy * dy + dz * dz));   // Eigen's norm of a 3-vector: x^2 + (y^2 + z^2)
    if ((double)dn > (double)res * 0.75) return type;
    double A[9], w[3], V[9];
    for (int k = 0; k < 9; k++) A[k] = (double)cov[k];
    jacobi_eig3(A, w, V);
    if (w[1] * (1.0 / 3.0) > w[0]) { type = PLANE; vec[0] = (float)V[0]; vec[1] = (float)V[3]; vec[2] = (float)V[6]; }
    else if (w[2] * (1.0 / 3.0) > w[1]) { type = LINE; vec[0] = (float)V[2]; vec[1] = (float)V[5]; vec[2] = (float)V[8]; }
    return type;
  }
};
typedef std::shared_ptr<Cell> CellPtr;

inline uint64_t pack_key(int k, int j, int i) {
  const int B = 1 << 20;
  return ((uint64_t)(unsigned)(k + B) << 42) | ((uint64_t)(unsigned)(j + B) << 21) | (uint64_t)(unsigned)(i + B);
}

// Points_cloud_map<float> as m_pt_cell_map_full uses it: append_cloud with cell_vec (:585-672), find_cell(pt, 1, 1) (:716-758)
struct CellMap {
  float res = 0.5f;   // set_resolution(r) stores r / 2
  int threshold = 2147483647, frame = 0;
  bool incremental = false;
  std::map<uint64_t, CellPtr> cells;

  CellPtr find_cell(const std::array<float, 3>& p) {
    const float box = res * 1.0f, half = res * 0.5f;
    const float fi = std::round((p[0] - half) / box), fj = std::round((p[1] - half) / box), fk = std::round((p[2] - half) / box);
    const int i = (int)fi, j = (int)fj, k = (int)fk;
    const uint64_t key = pack_key(k, j, i);
    auto it = cells.find(key);
    if (it == cells.end()) {   // add_cell: the map's incremental flag (:699)
      CellPtr c = std::make_shared<Cell>();
      c->key = key; c->res = res; c->incremental = incremental;
      c->center[0] = fi * box + half; c->center[1] = fj * box + half; c->center[2] = fk * box + half;
      c->inc = 0; last_update[key] = frame;
      cells[key] = c; return c;
    }
    if (frame - last_update[key] < threshold) { last_update[key] = frame; return it->second; }
    CellPtr c = std::make_shared<Cell>(*it->second);   // revisit: a new, empty cell without the map's flag (:747-752)
    c->pts.clear(); for (int q = 0; q < 3; q++) { c->xyz_sum[q] = 0.f; c->mean[q] = 0.f; } for (float& v : c->cov) v = 0.f;
    c->incremental = false; c->inc = it->second->inc + 1; c->type = SPHERE;
    last_update[key] = frame; it->second = c;
    return c;
  }
  // cell_vec: the cells of this call as add_cells receives them
  void append_cloud(const std::vector<std::array<float, 3>>& in, std::vector<CellPtr>* cell_vec) {
    const bool first = cells.empty();
    std::map<Cell*, std::pair<CellPtr, int>> seen;
    for (const auto& p : in) {
      if (!(std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]))) continue;
      CellPtr c = find_cell(p);
      c->append_pt(p);
      auto& e = seen[c.get()]; e.first = c; e.second++;
    }
    if (cell_vec) { cell_vec->clear(); for (auto& kv : seen) if (first || kv.second.second >= 3) cell_vec->push_back(kv.second.first); }
    if (first) frame++;
    frame++;
  }
  std::map<uint64_t, int> last_update;
};

// cv::getGaussianKernel(9, 4, CV_32F) and GaussianBlur on the image wrap-padded by 5, cropped (apply_guassian_blur(img, 4, 4), :1358-1370):
// with the pad wider than the radius the crop is a circular separable convolution, rows (x) first, float sums in tap order.
inline void gaussian_kernel(float k[9]) {
  double t[9], s = 0.0;
  for (int i = 0; i < 9; i++) { const double x = i - 4.0; t[i] = std::exp(-x * x / (2.0 * 16.0)); s += t[i]; }
  for (int i = 0; i < 9; i++) k[i] = (float)(t[i] / s);
}
inline void blur(const float* in, float* out) {
  float k[9]; gaussian_kernel(k);
  std::vector<float> tmp(PIX);
  for (int r = 0; r < RES; r++) for (int c = 0; c < RES; c++) {
    float s = 0.f; for (int t = 0; t < 9; t++) s = s + k[t] * in[r * RES + (c + t - 4 + RES) % RES]; tmp[r * RES + c] = s;
  }
  for (int r = 0; r < RES; r++) for (int c = 0; c < RES; c++) {
    float s = 0.f; for (int t = 0; t < 9; t++) s = s + k[t] * tmp[((r + t - 4 + RES) % RES) * RES + c]; out[r * RES + c] = s;
  }
}
inline float ratio_nonzero(const float* img) { int n = 0; for (int p = 0; p < PIX; p++) n += img[p] >= 1.0f; return (float)n / (float)PIX; }

// max_similiarity_of_two_image(a, b) (:1157-1229): matchTemplate(add_padding_to_feature_image(b, 30, 30), a, CV_TM_CCORR_NORMED), max of the
// 61 x 61 result.  Sums in float, row-major; OpenCV's normalisation in double: num / t if |num| < t, +-1 if |num| < 1.125 t, else 0.
inline float max_similarity(const float* a, const float* b) {
  const int W = RES + 60;
  std::vector<float> P(W * W);
  for (int r = 0; r < W; r++) for (int c = 0; c < W; c++) P[r * W + c] = b[((r + 30) % RES) * RES + (c + 30) % RES];
  float tn = 0.f; for (int p = 0; p < PIX; p++) tn = tn + a[p] * a[p];
  float best = 0.f; bool any = false;
  for (int y = 0; y <= 60; y++) for (int x = 0; x <= 60; x++) {
    float num = 0.f, den = 0.f;
    for (int r = 0; r < RES; r++) for (int c = 0; c < RES; c++) { const float v = P[(y + r) * W + x + c]; num = num + a[r * RES + c] * v; den = den + v * v; }
    const double t = std::sqrt((double)den * (double)tn);
    double v = num;
    if (std::fabs(v) < t) v = v / t; else if (std::fabs(v) < t * 1.125) v = v > 0 ? 1.0 : -1.0; else v = 0.0;
    const float fv = (float)v;
    if (!any || fv > best) { best = fv; any = true; }
  }
  return best;
}

// Maps_keyframe<float>
struct Keyframe {
  std::map<std::pair<uint64_t, int>, CellPtr> cells;   // (key, incarnation): the pinned order of m_set_cell
  unsigned accumulate_frames = 0;
  float center[3] = {0, 0, 0}, roi_range = 0.f, ratio_line = 0.f, ratio_plane = 0.f;
  std::vector<float> count_line = std::vector<float>(PIX), count_plane = std::vector<float>(PIX), img_line = std::vector<float>(PIX), img_plane = std::vector<float>(PIX);

  void add_cells(const std::vector<CellPtr>& v) { for (const CellPtr& c : v) cells[{c->key, c->inc}] = c; accumulate_frames++; }   // :1243-1261

  static void bin(float x, float y, float z, int& pi, int& ti) {   // feature_direction (:1073-1090)
    if (x < 0) { x = -x; y = -y; z = -z; }
    const double step = M_PI / RES;
    // atan2 / asin of float arguments are the float overloads (using namespace std); pinned to (float) of the double functions
    const double phi = (double)(float)std::atan2((double)y, (double)x) + M_PI / 2, theta = (double)(float)std::asin((double)z) + M_PI / 2;
    const double fp = std::floor(phi / step), ft = std::floor(theta / step);
    pi = fp != fp ? 0 : (fp < 0 ? 0 : (fp >= RES ? RES - 1 : (int)fp));
    ti = ft != ft ? 0 : (ft < 0 ? 0 : (ft >= RES ? RES - 1 : (int)ft));
  }
  void analyze() {   // :1487-1494 (the ROI images are not built: their only reader is disabled, laser_mapping.hpp:1015)
    for (auto& kv : cells) kv.second->determine_feature();
    std::fill(count_line.begin(), count_line.end(), 0.f); std::fill(count_plane.begin(), count_plane.end(), 0.f);
    roi_range = 0.f; center[0] = center[1] = center[2] = 0.f;
    if (cells.empty()) { blur(count_line.data(), img_line.data()); blur(count_plane.data(), img_plane.data()); ratio_line = ratio_plane = 0.f; return; }
    float c[3] = {0, 0, 0};
    for (auto& kv : cells) for (int a = 0; a < 3; a++) c[a] = c[a] + kv.second->center[a];
    const float f = (float)(1.0 / (double)(float)cells.size());
    for (int a = 0; a < 3; a++) center[a] = c[a] * f;
    std::set<float> dis;
    for (auto& kv : cells) {
      const float dx = kv.second->center[0] - center[0], dy = kv.second->center[1] - center[1], dz = kv.second->center[2] - center[2];
      dis.insert(std::sqrt(dx * dx + (dy * dy + dz * dz)));
    }
    roi_range = *std::next(dis.begin(), (long)std::ceil((float)(dis.size() - 1) * 0.9f));
    double M[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    for (auto& kv : cells) if (kv.second->type == PLANE) {
      const float* q = kv.second->vec;
      for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) M[a * 3 + b] = M[a * 3 + b] + (double)(q[a] * q[b]);
    }
    double w[3], V[9];
    jacobi_eig3(M, w, V);
    const float R0[3] = {(float)V[2], (float)V[5], (float)V[8]}, R1[3] = {(float)V[1], (float)V[4], (float)V[7]};
    const float R2[3] = {R0[1] * R1[2] - R0[2] * R1[1], R0[2] * R1[0] - R0[0] * R1[2], R0[0] * R1[1] - R0[1] * R1[0]};
    auto dot = [](const float* a, const float* b) { return a[0] * b[0] + (a[1] * b[1] + a[2] * b[2]); };
    for (auto& kv : cells) {
      const int t = kv.second->type;
      if (t != LINE && t != PLANE) continue;
      const float* q = kv.second->vec;
      int pi, ti; bin(dot(R0, q), dot(R1, q), dot(R2, q), pi, ti);
      (t == LINE ? count_line : count_plane)[pi * RES + ti] += 1.f;
    }
    ratio_line = ratio_nonzero(count_line.data()); ratio_plane = ratio_nonzero(count_plane.data());
    blur(count_line.data(), img_line.data()); blur(count_plane.data(), img_plane.data());
  }
  // extract_specify_points(type) / get_all_pointcloud() (type < 0)
  std::vector<std::array<float, 3>> cloud(int type) const {
    std::vector<std::array<float, 3>> out;
    for (auto& kv : cells) if (type < 0 || kv.second->type == type) out.insert(out.end(), kv.second->pts.begin(), kv.second->pts.end());
    return out;
  }
};

struct LoopCfg { int minimum_keyframe_differen = 200; float avail_ratio_plane = 0.05f, avail_ratio_line = 0.03f, maximum_roi_difference = 5.0f;
                 float minimum_similarity_linear = 0.65f, minimum_similarity_planar = 0.94f; double plane_with_line = 0.92; };
struct KfSummary { size_t cells; float roi_range, ratio_plane, ratio_line; };

// laser_mapping.hpp:994-1033 for keyframe `newest` against `his`, given the two similarities: true when the pair goes on to scene alignment
inline bool loop_gates(const LoopCfg& g, size_t n_keyframes, size_t his, const KfSummary& last, const KfSummary& old, float sim_plane, float sim_line) {
  if (n_keyframes - his < (size_t)g.minimum_keyframe_differen) return false;
  if (old.ratio_plane < g.avail_ratio_plane && old.ratio_line < g.avail_ratio_line) return false;
  if (std::abs(old.roi_range - last.roi_range) > (double)g.maximum_roi_difference) return false;
  if (!((sim_line > g.minimum_similarity_linear && sim_plane > g.plane_with_line) || sim_plane > g.minimum_similarity_planar)) return false;
  if (last.cells + old.cells == 0) return false;
  if ((last.cells - old.cells) / (last.cells + old.cells) * 0.1) return false;
  return true;
}

}  // namespace orc_kf
