// Compiled, linked against libloamlivox_b200.so and run by tests/test_keyframe_oracle.py (no GPU needed to build; without a GPU the run stops
// at the context).  Maps_keyframe over a full-resolution Points_cloud_map: append, analyze, typed clouds, centre, similarity and the search.
#include <cmath>
#include <cstdio>
#include "loamlivox_b200.hpp"

static ll200::PointCloud corner(float shift, unsigned seed) {
  ll200::PointCloud c;
  auto rnd = [&seed]() { seed = seed * 1664525u + 1013904223u; return (seed >> 8) * (1.0f / 16777216.0f); };
  auto push = [&c](float x, float y, float z) { ll200::PointXYZI p{}; p.x = x; p.y = y; p.z = z; p._pad0 = 1.f; c.push_back(p); };
  for (int i = 0; i < 20000; i++) push(8 * rnd() + shift, 6 * rnd(), 0.02f * (rnd() - 0.5f));          // floor
  for (int i = 0; i < 10000; i++) push(shift + 0.02f * (rnd() - 0.5f), 6 * rnd(), 3 * rnd());           // wall
  for (int i = 0; i < 3000; i++) push(2.1f + shift + 0.02f * (rnd() - 0.5f), 3.1f + 0.02f * (rnd() - 0.5f), 3 * rnd());   // pole
  return c;
}

int main() {
  if (ll_keyframe_create(nullptr, nullptr) != LL_ERR_INVALID) return 2;
  if (ll_loop_search(nullptr, nullptr, 0, 0, nullptr, nullptr, nullptr, nullptr, nullptr) != LL_ERR_INVALID) return 2;
  ll_loop_cfg cfg; ll_loop_cfg_default(&cfg);
  if (cfg.minimum_keyframe_differen != 200 || cfg.plane_with_line != 0.92) return 2;
  try {
    ll200::Context ctx(0);
    ll200::Points_cloud_map full(ctx, 1.0f, 2147483647);
    ll200::Maps_keyframe a(ctx), b(ctx);
    ll200::Maps_keyframe::append_cloud(ctx, full, corner(0.f, 1), {&a});
    ll200::Maps_keyframe::append_cloud(ctx, full, corner(0.05f, 2), {&a, &b});
    a.analyze(full); b.analyze(full);
    const ll200::PointCloud pl = a.extract_specify_points(ll200::e_feature_plane), li = a.extract_specify_points(ll200::e_feature_line);
    const ll200::PointCloud all = a.get_all_pointcloud();
    if (pl.size() != a.info().plane_points || li.size() != a.info().line_points || all.size() != a.info().all_points || pl.empty()) return 3;
    const std::array<float, 3> c = a.get_center();
    if (!(std::isfinite(c[0]) && c[0] > 0.f)) return 4;
    const float s = ll200::Maps_keyframe::max_similiarity_of_two_image(ctx, b, a, ll200::e_feature_plane);
    if (!(s > 0.5f && s <= 1.f)) return 5;
    cfg.minimum_keyframe_differen = 1;
    const std::vector<int> cand = ll200::loop_search(ctx, {&a, &b}, 1, cfg);
    std::printf("GPU run: %d cells, %zu plane / %zu line points, plane similarity %.4f, %zu candidate(s)\n", a.info().cells, pl.size(), li.size(), s, cand.size());
  } catch (const ll200::Error& err) {
    if (err.status != LL_ERR_CUDA) { std::printf("unexpected status %d\n", err.status); return 6; }
    std::printf("no GPU: context refused (LL_ERR_CUDA), as it must -- there is no CPU fallback\n");
  }
  return 0;
}
