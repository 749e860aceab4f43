// Compiled, linked against libloamlivox_b200.so and run by tests/test_loop_feedback.py (no GPU needed to build; without a GPU the run stops at
// the context).  With the argument "layout" it prints the loop-feedback constants and sizeof(ll_pose) for the ctypes mirrors.  Otherwise
// ll_loop_correction on the host, then the C++ mirror's set_loop_feedback / loop_correction: refused without loop closure and in matching
// mode 1, accepted in mode 0, and a version-3 loop image saved and restored on a second context.
#include <cmath>
#include <cstdio>
#include <cstring>
#include "loamlivox_b200.hpp"

static int layout() {
  std::printf("const LL_LOOP_IMAGE_VERSION_FEEDBACK %d\n", LL_LOOP_IMAGE_VERSION_FEEDBACK);
  std::printf("const LL_LOOP_IMAGE_FEEDBACK %d\n", (int)LL_LOOP_IMAGE_FEEDBACK);
  std::printf("const LL_LOOP_IMAGE_SECTIONS %d\n", (int)LL_LOOP_IMAGE_SECTIONS);
  std::printf("const LL_LOOP_IMAGE_SECTIONS_FEEDBACK %d\n", (int)LL_LOOP_IMAGE_SECTIONS_FEEDBACK);
  std::printf("const LL_LOOP_FEEDBACK_MAX_SEGMENTS %d\n", LL_LOOP_FEEDBACK_MAX_SEGMENTS);
  std::printf("sizeof ll_pose %zu\n", sizeof(ll_pose));
  return 0;
}

static bool refused(ll200::Laser_mapping& m, bool on) {
  try { m.set_loop_feedback(on); return false; } catch (const ll200::Error& e) { return e.status == LL_ERR_INVALID; }
}

int main(int argc, char** argv) {
  if (argc > 1 && std::strcmp(argv[1], "layout") == 0) return layout();
  // the rule: keyframe 1 turned by 90 degrees about z and moved; halfway between frames 10 and 20 the correction turns by 45 degrees
  ll_pose ori[2] = {{{1, 0, 0, 0}, {0, 0, 0}}, {{1, 0, 0, 0}, {1, 0, 0}}};
  ll_pose opt[2] = {{{1, 0, 0, 0}, {0, 0, 0}}, {{std::sqrt(0.5), 0, 0, std::sqrt(0.5)}, {1, 1, 0}}};
  const int f[2] = {10, 20};
  double q[4], t[3];
  if (ll_loop_correction(ori, opt, f, 2, 15, q, t) != LL_OK) return 2;
  if (std::fabs(q[0] - std::cos(M_PI / 8)) > 1e-12 || std::fabs(q[3] - std::sin(M_PI / 8)) > 1e-12) { std::printf("slerp off\n"); return 2; }
  if (ll_loop_correction(ori, opt, f, 2, 5, q, t) != LL_OK || q[0] != 1.0 || t[0] != 0.0) return 2;
  const int bad[2] = {20, 10};
  if (ll_loop_correction(ori, opt, bad, 2, 15, q, t) != LL_ERR_INVALID) return 2;
  if (ll_mapper_set_loop_feedback(nullptr, 1) != LL_ERR_INVALID) return 2;
  try {
    ll200::Context ctx(0), other(0);
    ll200::Laser_mapping mapping(ctx);
    if (!refused(mapping, true)) { std::printf("feedback accepted with loop closure off\n"); return 3; }
    ll_loop_closure_cfg cfg; ll_mapper_loop_closure_default(&cfg);
    cfg.scans_of_each_keyframe = 3; cfg.scans_between_two_keyframe = 1; cfg.reserve_map_points = 1 << 16; cfg.reserve_history_points = 1 << 16; cfg.reserve_keyframes = 8;
    mapping.set_loop_closure(&cfg);
    mapping.set_loop_feedback(true);
    if (mapping.loop_correction(q, t) != 0 || q[0] != 1.0) { std::printf("a correction before a loop\n"); return 4; }
    ll200::PointCloud raw(200);
    for (size_t i = 0; i < raw.size(); i++) { raw[i].x = 5.f; raw[i].y = 0.01f * i; raw[i].z = 0.f; raw[i].intensity = 10.f; }
    for (int k = 0; k < 5; k++) mapping.process_new_scan(raw, 100.0 + 0.1 * k);
    std::vector<uint8_t> image, loop, again;
    mapping.save_to_image(image);
    mapping.loop_save(loop);
    ll_loop_image_summary info;
    if (ll_loop_image_info(loop.data(), loop.size(), &info) != LL_OK || info.version != LL_LOOP_IMAGE_VERSION_FEEDBACK) { std::printf("not a version-3 image\n"); return 5; }
    std::unique_ptr<ll200::Laser_mapping> restored = ll200::Laser_mapping::load_from_image(other, image);
    restored->loop_load(loop);
    restored->loop_save(again);
    if (again != loop) { std::printf("restored loop image differs\n"); return 6; }
    ll_mapper_config mc; ll_mapper_config_default(&mc); mc.matching_mode = 1;
    ll200::Laser_mapping cells(ctx, &mc);
    cells.set_loop_closure(&cfg);
    if (!refused(cells, true)) { std::printf("feedback accepted in matching mode 1\n"); return 7; }
    std::printf("GPU run: version-3 loop image of %zu bytes\n", loop.size());
  } catch (const ll200::Error& e) {
    if (e.status != LL_ERR_CUDA) { std::printf("unexpected status %d\n", e.status); return 8; }
    std::printf("no GPU: context refused (LL_ERR_CUDA), as it must -- there is no CPU fallback\n");
  }
  return 0;
}
