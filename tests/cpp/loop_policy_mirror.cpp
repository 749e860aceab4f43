// Compiled, linked against libloamlivox_b200.so and run by tests/test_loop_policy.py (no GPU needed to build; without a GPU the run stops at the
// context).  With the argument "layout" it prints sizeof / offsetof of ll_loop_policy and the policy's constants as "name field value" lines
// for the ctypes mirrors.  Otherwise the C++ mirror's set_loop_policy / loop_edges: the default, refusals without loop closure and out of
// range, a multi-loop policy on a tiny stream, and a loop image of version 2 saved and restored on a second context.
#include <cstddef>
#include <cstdio>
#include <cstring>
#include "loamlivox_b200.hpp"

static int layout() {
  std::printf("ll_loop_policy sizeof %zu\n", sizeof(ll_loop_policy));
  std::printf("ll_loop_policy max_loops %zu\n", offsetof(ll_loop_policy, max_loops));
  std::printf("ll_loop_policy min_keyframes_between_loops %zu\n", offsetof(ll_loop_policy, min_keyframes_between_loops));
  std::printf("const LL_MAX_LOOPS %d\n", LL_MAX_LOOPS);
  std::printf("const LL_LOOP_IMAGE_VERSION_POLICY %d\n", LL_LOOP_IMAGE_VERSION_POLICY);
  return 0;
}

int main(int argc, char** argv) {
  if (argc > 1 && std::strcmp(argv[1], "layout") == 0) return layout();
  ll_loop_policy p; std::memset(&p, 0xff, sizeof(p));
  ll_mapper_loop_policy_default(&p);
  if (p.max_loops != 1 || p.min_keyframes_between_loops != 0) return 2;
  ll_mapper_loop_policy_default(nullptr);   // (no effect, no fault)
  int n = 0;
  if (ll_mapper_set_loop_policy(nullptr, &p) != LL_ERR_INVALID || ll_mapper_loop_edges(nullptr, nullptr, 0, &n) != LL_ERR_INVALID) return 2;
  try {
    ll200::Context ctx(0), other(0);
    ll200::Laser_mapping mapping(ctx);
    ll_loop_policy multi{4, 2};
    try { mapping.set_loop_policy(&multi); std::printf("policy accepted with loop closure off\n"); return 3; } catch (const ll200::Error& e) {
      if (e.status != LL_ERR_INVALID) return 3;
    }
    ll_loop_closure_cfg cfg; ll_mapper_loop_closure_default(&cfg);
    cfg.scans_of_each_keyframe = 3; cfg.scans_between_two_keyframe = 1; cfg.reserve_map_points = 1 << 16; cfg.reserve_history_points = 1 << 16; cfg.reserve_keyframes = 8;
    mapping.set_loop_closure(&cfg);
    ll_loop_policy bad{LL_MAX_LOOPS + 1, 0};
    try { mapping.set_loop_policy(&bad); std::printf("max_loops above LL_MAX_LOOPS accepted\n"); return 4; } catch (const ll200::Error& e) {
      if (e.status != LL_ERR_INVALID) return 4;
    }
    mapping.set_loop_policy(&multi);
    ll200::PointCloud raw(200);
    for (size_t i = 0; i < raw.size(); i++) { raw[i].x = 5.f; raw[i].y = 0.01f * i; raw[i].z = 0.f; raw[i].intensity = 10.f; }
    for (int k = 0; k < 5; k++) mapping.process_new_scan(raw, 100.0 + 0.1 * k);
    if (!mapping.loop_edges().empty()) { std::printf("a loop edge without a loop\n"); return 5; }
    std::vector<uint8_t> image, loop, again;
    mapping.save_to_image(image);
    mapping.loop_save(loop);
    ll_loop_image_summary info;
    if (ll_loop_image_info(loop.data(), loop.size(), &info) != LL_OK || info.version != LL_LOOP_IMAGE_VERSION_POLICY) { std::printf("not a version-2 image\n"); return 6; }
    std::unique_ptr<ll200::Laser_mapping> restored = ll200::Laser_mapping::load_from_image(other, image);
    restored->loop_load(loop);
    restored->loop_save(again);
    if (again != loop) { std::printf("restored loop image differs\n"); return 7; }
    std::printf("GPU run: version-2 loop image of %zu bytes\n", loop.size());
  } catch (const ll200::Error& e) {
    if (e.status != LL_ERR_CUDA) { std::printf("unexpected status %d\n", e.status); return 8; }
    std::printf("no GPU: context refused (LL_ERR_CUDA), as it must -- there is no CPU fallback\n");
  }
  return 0;
}
