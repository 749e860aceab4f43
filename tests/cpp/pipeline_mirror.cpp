// Compiled, linked against libloamlivox_b200.so and run by tests/test_pipeline_cabi.py (no GPU needed to build; without a GPU the run stops at
// the context).  Laser_mapping::process_new_frames / process_new_scans of the C++ mirror on a few tiny frames.
#include <cstdio>
#include "loamlivox_b200.hpp"

int main() {
  int done = -1, n_pieces[1];
  ll_reg_result r[1]; ll_mapper_stats s[1];
  if (ll_mapper_process_frames(nullptr, 1, 1, nullptr, nullptr, LL_FMT_PCL32, LL_HOST, nullptr, 1, r, s, 1, n_pieces, &done) != LL_ERR_INVALID) return 2;
  if (ll_mapper_process_scans(nullptr, 1, nullptr, nullptr, LL_FMT_PCL32, LL_HOST, nullptr, r, s, &done) != LL_ERR_INVALID) return 2;
  try {
    ll200::Context ctx(0);
    ll200::Laser_mapping mapping(ctx);
    ll200::PointCloud raw(200);
    for (size_t i = 0; i < raw.size(); i++) { raw[i].x = 5.f; raw[i].y = 0.01f * i; raw[i].z = 0.f; raw[i].intensity = 10.f; }
    std::vector<std::vector<ll_reg_result>> fr;
    mapping.process_new_frames({{raw}, {raw}}, {{100.0}, {100.1}}, 1, &fr);   // a few petals: nothing published
    std::vector<int> st = mapping.process_new_scans({raw, raw}, {100.2, 100.3});
    if (fr.size() != 2 || st.size() != 2) { std::printf("unexpected sequence result\n"); return 3; }
    std::printf("GPU run: %zu + %zu pieces, frame index %d\n", fr[0].size(), fr[1].size(), mapping.m_current_frame_index);
  } catch (const ll200::Error& e) {
    if (e.status != LL_ERR_CUDA) { std::printf("unexpected status %d\n", e.status); return 5; }
    std::printf("no GPU: context refused (LL_ERR_CUDA), as it must -- there is no CPU fallback\n");
  }
  return 0;
}
