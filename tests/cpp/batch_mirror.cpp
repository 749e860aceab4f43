// Compiled, linked against libloamlivox_b200.so and run by tests/test_batch_cabi.py (no GPU needed to build; without a GPU the run stops at the
// context).  Point_cloud_registration::register_batch of the C++ mirror: two items, one scan shared by both.
#include <cstdio>
#include "loamlivox_b200.hpp"

int main() {
  static_assert(LL_MAX_BATCH == 16, "LL_MAX_BATCH");
  if (ll_register_batch(nullptr, nullptr, 1, nullptr, nullptr, nullptr, nullptr, LL_FMT_PCL32, LL_HOST, nullptr, nullptr, nullptr) != LL_ERR_INVALID) return 2;
  try {
    ll200::Context ctx(0);
    ll200::PointCloud corner(40), surf(400);
    for (size_t i = 0; i < corner.size(); i++) { corner[i].x = 3.f; corner[i].y = 1.f; corner[i].z = 0.05f * i; }
    for (size_t i = 0; i < surf.size(); i++) { surf[i].x = 0.05f * (i % 20); surf[i].y = 0.05f * (i / 20); surf[i].z = 0.f; }
    ll200::Match_map map(ctx, corner, surf);
    ll200::Point_cloud_registration reg(ctx);
    ll_reg_state s[2]; ll_reg_state_default(&s[0]); ll_reg_state_default(&s[1]);
    s[1].current_frame_index = 0;   // under the :199 gate: returns unregistered
    std::vector<ll_reg_result> r; std::vector<int> st;
    reg.register_batch(map, {{&corner, &surf}, {&corner, &surf}}, {s[0], s[1]}, r, st);
    if (r.size() != 2 || st[1] != LL_OK || r[1].registered != 0) { std::printf("unexpected batch result\n"); return 3; }
    std::printf("GPU run: item 0 status %d, %d ICP iterations\n", st[0], r[0].icp_iterations);
  } catch (const ll200::Error& e) {
    if (e.status != LL_ERR_CUDA) { std::printf("unexpected status %d\n", e.status); return 5; }
    std::printf("no GPU: context refused (LL_ERR_CUDA), as it must -- there is no CPU fallback\n");
  }
  return 0;
}
