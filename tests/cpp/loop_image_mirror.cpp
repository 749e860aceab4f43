// Compiled, linked against libloamlivox_b200.so and run by tests/test_loop_image.py (no GPU needed to build; without a GPU the run stops at the
// context).  With the argument "layout" it prints sizeof / offsetof of the loop image's structs as "struct field value" lines for the ctypes
// mirrors.  Otherwise Laser_mapping::loop_save / loop_load of the C++ mirror: a tiny stream with loop closure on, both images saved, both loaded
// on a second context, and the restored mapper's loop image equal to the saved one.
#include <cstddef>
#include <cstdio>
#include <cstring>
#include "loamlivox_b200.hpp"

#define F(T, f) std::printf(#T " " #f " %zu\n", offsetof(T, f))
static int layout() {
  std::printf("ll_loop_image_header sizeof %zu\n", sizeof(ll_loop_image_header));
  std::printf("ll_loop_image_scalars sizeof %zu\n", sizeof(ll_loop_image_scalars));
  F(ll_loop_image_scalars, frame_index); F(ll_loop_image_scalars, matching_mode); F(ll_loop_image_scalars, threshold_cell_revisit);
  F(ll_loop_image_scalars, maximum_history_size); F(ll_loop_image_scalars, pieces); F(ll_loop_image_scalars, cell_resolution);
  F(ll_loop_image_scalars, last_time_stamp); F(ll_loop_image_scalars, q_w_curr); F(ll_loop_image_scalars, t_w_curr); F(ll_loop_image_scalars, closed);
  F(ll_loop_image_scalars, stopped); F(ll_loop_image_scalars, n_keyframes); F(ll_loop_image_scalars, n_open); F(ll_loop_image_scalars, n_events);
  F(ll_loop_image_scalars, n_dropped);
  std::printf("ll_loop_image_summary sizeof %zu\n", sizeof(ll_loop_image_summary));
  F(ll_loop_image_summary, bytes); F(ll_loop_image_summary, cells); F(ll_loop_image_summary, cell_points); F(ll_loop_image_summary, replaced_points);
  F(ll_loop_image_summary, history_points); F(ll_loop_image_summary, cloud_points); F(ll_loop_image_summary, accumulated_points);
  F(ll_loop_image_summary, version); F(ll_loop_image_summary, frame_index); F(ll_loop_image_summary, matching_mode); F(ll_loop_image_summary, closed);
  F(ll_loop_image_summary, stopped); F(ll_loop_image_summary, keyframes); F(ll_loop_image_summary, open_keyframes); F(ll_loop_image_summary, events);
  F(ll_loop_image_summary, dropped); F(ll_loop_image_summary, max_incarnation);
  std::printf("ll_loop_image_open sizeof %zu\n", sizeof(ll_loop_image_open));
  std::printf("ll_loop_image_ref sizeof %zu\n", sizeof(ll_loop_image_ref));
  std::printf("ll_keyframe_info sizeof %zu\n", sizeof(ll_keyframe_info));
  std::printf("ll_pose sizeof %zu\n", sizeof(ll_pose));
  std::printf("ll_pg_edge sizeof %zu\n", sizeof(ll_pg_edge));
  return 0;
}

int main(int argc, char** argv) {
  if (argc > 1 && std::strcmp(argv[1], "layout") == 0) return layout();
  ll_loop_image_summary info;
  if (ll_loop_image_info(nullptr, 0, &info) != LL_ERR_INVALID) return 2;   // host-only validation needs no context
  size_t n = 0;
  if (ll_mapper_loop_save(nullptr, nullptr, 0, &n) != LL_ERR_INVALID || ll_mapper_loop_load(nullptr, nullptr, 0, nullptr) != LL_ERR_INVALID) return 2;
  try {
    ll200::Context ctx(0), other(0);
    ll200::Laser_mapping mapping(ctx);
    ll_loop_closure_cfg cfg; ll_mapper_loop_closure_default(&cfg);
    cfg.scans_of_each_keyframe = 3; cfg.scans_between_two_keyframe = 1; cfg.reserve_map_points = 1 << 16; cfg.reserve_history_points = 1 << 16; cfg.reserve_keyframes = 8;
    mapping.set_loop_closure(&cfg);
    ll200::PointCloud raw(200);
    for (size_t i = 0; i < raw.size(); i++) { raw[i].x = 5.f; raw[i].y = 0.01f * i; raw[i].z = 0.f; raw[i].intensity = 10.f; }
    for (int k = 0; k < 4; k++) mapping.process_new_scan(raw, 100.0 + 0.1 * k);
    std::vector<uint8_t> image, loop, again;
    mapping.save_to_image(image);
    mapping.loop_save(loop);
    std::unique_ptr<ll200::Laser_mapping> restored = ll200::Laser_mapping::load_from_image(other, image);
    restored->loop_load(loop);
    restored->loop_save(again);
    if (again != loop) { std::printf("restored loop image differs\n"); return 3; }
    std::printf("GPU run: loop image of %zu bytes\n", loop.size());
  } catch (const ll200::Error& e) {
    if (e.status != LL_ERR_CUDA) { std::printf("unexpected status %d\n", e.status); return 5; }
    std::printf("no GPU: context refused (LL_ERR_CUDA), as it must -- there is no CPU fallback\n");
  }
  return 0;
}
