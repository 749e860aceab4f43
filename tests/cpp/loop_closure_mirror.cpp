// Compiled and linked against libloamlivox_b200.so by tests/test_loop_closure_cabi.py (no GPU needed to build; without a GPU the run stops at
// the context).  The loop-closure calls of the C API and Laser_mapping::set_loop_closure / loop_log / loop_result of the C++ mirror.
#include <cstdio>
#include "loamlivox_b200.hpp"

int main() {
  ll_loop_closure_cfg cfg; ll_mapper_loop_closure_default(&cfg);
  ll_loop_event e[1]; int n = -1, dropped = -1, closed = -1; size_t np = 0;
  if (ll_mapper_set_loop_closure(nullptr, &cfg) != LL_ERR_INVALID || ll_mapper_loop_read(nullptr, e, 1, &n, &dropped) != LL_ERR_INVALID) return 2;
  if (ll_mapper_loop_result(nullptr, &n, &closed, nullptr, nullptr, 0, nullptr) != LL_ERR_INVALID) return 2;
  if (ll_mapper_loop_cloud(nullptr, 0, nullptr, 0, &np, nullptr) != LL_ERR_INVALID) return 2;
  try {
    ll200::Context ctx(0);
    ll200::Laser_mapping mapping(ctx);
    cfg.scans_of_each_keyframe = 3; cfg.scans_between_two_keyframe = 1;
    mapping.set_loop_closure(&cfg);
    ll200::PointCloud raw(200);
    for (size_t i = 0; i < raw.size(); i++) { raw[i].x = 5.f; raw[i].y = 0.01f * i; raw[i].z = 0.f; raw[i].intensity = 10.f; }
    mapping.process_new_scans({raw, raw, raw, raw}, {100.0, 100.1, 100.2, 100.3});
    int d = 0;
    const std::vector<ll_loop_event> log = mapping.loop_log(&d);
    std::vector<ll_pose> ori, opt;
    const bool c = mapping.loop_result(&ori, &opt);
    mapping.set_loop_closure(nullptr);
    std::printf("GPU run: %zu events, %d dropped, %zu keyframes, closed %d\n", log.size(), d, ori.size(), (int)c);
  } catch (const ll200::Error& err) {
    if (err.status != LL_ERR_CUDA) { std::printf("unexpected status %d\n", err.status); return 5; }
    std::printf("no GPU: context refused (LL_ERR_CUDA), as it must -- there is no CPU fallback\n");
  }
  return 0;
}
