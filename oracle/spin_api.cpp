// ORACLE — TEST INFRASTRUCTURE ONLY. C entry points (ctypes) over orc_spin.hpp, the restatement of the reference's Velodyne front end.
#include <chrono>
#include <cstring>
#include "orc_spin.hpp"

using namespace orc;

extern "C" {

void* orc_spin_create(int scan_line, float minimum_range, float plane_resolution) {
  SpinExtractor* e = new SpinExtractor();
  e->scan_line = scan_line; e->minimum_range = minimum_range; e->plane_resolution = plane_resolution;
  return e;
}
void orc_spin_free(void* h) { delete (SpinExtractor*)h; }
// Returns the seconds the extraction took (one thread); counts[5]: full, sharp, less sharp, flat, less flat.
double orc_spin_extract(void* h, const float* raw4, int n, int* counts) {
  SpinExtractor* e = (SpinExtractor*)h;
  const auto t0 = std::chrono::steady_clock::now();
  e->extract(raw4, n);
  const double dt = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  counts[0] = (int)e->cloud.size(); counts[1] = (int)e->sharp.size(); counts[2] = (int)e->less_sharp.size();
  counts[3] = (int)e->flat.size(); counts[4] = (int)e->less_flat.size();
  return dt;
}
void orc_spin_cloud(void* h, int which, float* out4) {
  SpinExtractor* e = (SpinExtractor*)h;
  const std::vector<SpinPt>* c[5] = {&e->cloud, &e->sharp, &e->less_sharp, &e->flat, &e->less_flat};
  if (!c[which]->empty()) std::memcpy(out4, c[which]->data(), c[which]->size() * 16);
}
void orc_spin_point_info(void* h, int* ring, float* curvature, int* picked, int* label) {
  SpinExtractor* e = (SpinExtractor*)h;
  const size_t N = e->cloud.size();
  for (size_t i = 0; i < N; i++) { ring[i] = e->ring[i]; curvature[i] = e->curvature[i]; picked[i] = e->picked_before[i]; label[i] = e->label[i]; }
}

}  // extern "C"
