// C entry points over oracle/orc_keyframe.hpp for the tests (ctypes); built by tests/keyframe_reference.py.
#include <cstring>
#include "../../oracle/orc_keyframe.hpp"

using namespace orc_kf;

struct KfoMap { CellMap map; std::vector<Keyframe> kfs; };

extern "C" {

void* kfo_create(float resolution, int threshold, int incremental) {
  KfoMap* m = new KfoMap(); m->map.res = resolution * 0.5f; m->map.threshold = threshold; m->map.incremental = incremental != 0;
  return m;
}
void kfo_release(void* h) { delete (KfoMap*)h; }
int kfo_new_keyframe(void* h) { KfoMap* m = (KfoMap*)h; m->kfs.emplace_back(); return (int)m->kfs.size() - 1; }
// pts: n x 4 floats (x, y, z, unused)
void kfo_append(void* h, const float* pts, int n, const int* open, int n_open) {
  KfoMap* m = (KfoMap*)h;
  std::vector<std::array<float, 3>> in(n);
  for (int i = 0; i < n; i++) in[i] = {pts[4 * i], pts[4 * i + 1], pts[4 * i + 2]};
  std::vector<CellPtr> cv;
  m->map.append_cloud(in, &cv);
  for (int k = 0; k < n_open; k++) m->kfs[open[k]].add_cells(cv);
}
int kfo_cell_count(void* h) { return (int)((KfoMap*)h)->map.cells.size(); }
void kfo_analyze(void* h, int k) { ((KfoMap*)h)->kfs[k].analyze(); }
// fo: center xyz, roi, ratio line, ratio plane; io: cells, line cells, plane cells, accumulate_frames
void kfo_info(void* h, int k, float* fo, int* io) {
  const Keyframe& kf = ((KfoMap*)h)->kfs[k];
  fo[0] = kf.center[0]; fo[1] = kf.center[1]; fo[2] = kf.center[2]; fo[3] = kf.roi_range; fo[4] = kf.ratio_line; fo[5] = kf.ratio_plane;
  int nl = 0, np = 0; for (auto& kv : kf.cells) { nl += kv.second->type == LINE; np += kv.second->type == PLANE; }
  io[0] = (int)kf.cells.size(); io[1] = nl; io[2] = np; io[3] = (int)kf.accumulate_frames;
}
void kfo_cells(void* h, int k, uint64_t* keys, int* inc, int* type, float* vec) {
  int r = 0;
  for (auto& kv : ((KfoMap*)h)->kfs[k].cells) {
    keys[r] = kv.first.first; inc[r] = kv.first.second; type[r] = kv.second->type;
    for (int a = 0; a < 3; a++) vec[3 * r + a] = kv.second->vec[a];
    r++;
  }
}
void kfo_images(void* h, int k, float* out) {   // count line, count plane, line, plane
  const Keyframe& kf = ((KfoMap*)h)->kfs[k];
  memcpy(out, kf.count_line.data(), PIX * 4); memcpy(out + PIX, kf.count_plane.data(), PIX * 4);
  memcpy(out + 2 * PIX, kf.img_line.data(), PIX * 4); memcpy(out + 3 * PIX, kf.img_plane.data(), PIX * 4);
}
// which: 1 line, 2 plane, -1 all; out n x 4 (cap points); returns the point count
int kfo_cloud(void* h, int k, int which, float* out, int cap) {
  const auto c = ((KfoMap*)h)->kfs[k].cloud(which);
  for (int i = 0; i < (int)c.size() && i < cap; i++) { out[4 * i] = c[i][0]; out[4 * i + 1] = c[i][1]; out[4 * i + 2] = c[i][2]; out[4 * i + 3] = 0.f; }
  return (int)c.size();
}
// one constructed cell: its points in append order, centre, half resolution and covariance mode -> type, feature vector, mean, covariance
int kfo_cell_type(const float* pts, int n, const float* center, float res, int incremental, float* vec, float* mean, float* cov) {
  Cell c; c.res = res; c.incremental = incremental != 0;
  for (int a = 0; a < 3; a++) c.center[a] = center[a];
  for (int i = 0; i < n; i++) c.append_pt({pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]});
  const int t = c.determine_feature();
  for (int a = 0; a < 3; a++) { vec[a] = c.vec[a]; mean[a] = c.mean[a]; }
  for (int a = 0; a < 9; a++) cov[a] = c.cov[a];
  return t;
}
void kfo_eig3(const double* A, double* w, double* V) { jacobi_eig3(A, w, V); }
void kfo_blur(const float* in, float* out) { blur(in, out); }
float kfo_similarity(const float* a, const float* b) { return max_similarity(a, b); }
void kfo_gaussian_kernel(float* k) { gaussian_kernel(k); }
// the search of laser_mapping.hpp:988-1033 for keyframe `newest` over summaries and images (plane, line per keyframe: n x 2 x PIX floats);
// writes the similarities (newest x 2: plane, line) and the candidates; returns their count
int kfo_search(const int64_t* cells, const float* roi, const float* ratio_plane, const float* ratio_line, const float* imgs, int newest, const int* icfg,
               const float* fcfg, const double* dcfg, float* sims, int* cand) {
  LoopCfg g; g.minimum_keyframe_differen = icfg[0];
  g.avail_ratio_plane = fcfg[0]; g.avail_ratio_line = fcfg[1]; g.maximum_roi_difference = fcfg[2]; g.minimum_similarity_linear = fcfg[3];
  g.minimum_similarity_planar = fcfg[4]; g.plane_with_line = dcfg[0];
  const KfSummary last = {(size_t)cells[newest], roi[newest], ratio_plane[newest], ratio_line[newest]};
  int nc = 0;
  for (int his = 0; his < newest; his++) {
    const float sp = max_similarity(imgs + (2 * newest) * PIX, imgs + (2 * his) * PIX);
    const float sl = max_similarity(imgs + (2 * newest + 1) * PIX, imgs + (2 * his + 1) * PIX);
    sims[2 * his] = sp; sims[2 * his + 1] = sl;
    const KfSummary old = {(size_t)cells[his], roi[his], ratio_plane[his], ratio_line[his]};
    if (loop_gates(g, (size_t)newest + 1, (size_t)his, last, old, sp, sl)) cand[nc++] = his;
  }
  return nc;
}
int kfo_gates(const int64_t* cells, const float* roi, const float* ratio_plane, const float* ratio_line, const float* sims, int newest, const int* icfg,
              const float* fcfg, const double* dcfg, int* cand) {
  LoopCfg g; g.minimum_keyframe_differen = icfg[0];
  g.avail_ratio_plane = fcfg[0]; g.avail_ratio_line = fcfg[1]; g.maximum_roi_difference = fcfg[2]; g.minimum_similarity_linear = fcfg[3];
  g.minimum_similarity_planar = fcfg[4]; g.plane_with_line = dcfg[0];
  const KfSummary last = {(size_t)cells[newest], roi[newest], ratio_plane[newest], ratio_line[newest]};
  int nc = 0;
  for (int his = 0; his < newest; his++) {
    const KfSummary old = {(size_t)cells[his], roi[his], ratio_plane[his], ratio_line[his]};
    if (loop_gates(g, (size_t)newest + 1, (size_t)his, last, old, sims[2 * his], sims[2 * his + 1])) cand[nc++] = his;
  }
  return nc;
}

}
