// Compiled, linked against libloamlivox_b200.so and run by tests/test_checkpoint_image.py (no GPU needed to build; without a GPU the run
// stops at the context).  Laser_mapping::save_to_image / load_from_image of the C++ mirror: a tiny stream, a save, a load on a second
// context, and the image of the restored mapper equal to the saved one.
#include <cstdio>
#include "loamlivox_b200.hpp"

int main() {
  ll_image_info info;
  if (ll_mapper_image_info(nullptr, 0, &info) != LL_ERR_INVALID) return 2;   // host-only validation needs no context
  size_t n = 0;
  if (ll_mapper_save(nullptr, nullptr, 0, &n) != LL_ERR_INVALID) return 2;
  try {
    ll200::Context ctx(0), other(0);
    ll200::Laser_mapping mapping(ctx);
    ll200::PointCloud raw(200);
    for (size_t i = 0; i < raw.size(); i++) { raw[i].x = 5.f; raw[i].y = 0.01f * i; raw[i].z = 0.f; raw[i].intensity = 10.f; }
    mapping.process_new_scan(raw, 100.0);
    std::vector<uint8_t> image, again;
    mapping.save_to_image(image);
    std::unique_ptr<ll200::Laser_mapping> restored = ll200::Laser_mapping::load_from_image(other, image);
    restored->save_to_image(again);
    if (again != image || restored->m_current_frame_index != mapping.m_current_frame_index) { std::printf("restored mapper differs\n"); return 3; }
    std::printf("GPU run: image of %zu bytes, frame index %d\n", image.size(), restored->m_current_frame_index);
  } catch (const ll200::Error& e) {
    if (e.status != LL_ERR_CUDA) { std::printf("unexpected status %d\n", e.status); return 5; }
    std::printf("no GPU: context refused (LL_ERR_CUDA), as it must -- there is no CPU fallback\n");
  }
  return 0;
}
