// Compiled, linked against libloamlivox_b200.so and run by tests/test_pose_graph_cabi.py (no GPU needed to build; without a GPU the run stops
// at the context).  Pose_graph::pose_graph_optimization, add_constrain_of_loop and refine_pointclouds of the C++ mirror on a tiny graph.
#include <cmath>
#include <cstdio>
#include "loamlivox_b200.hpp"

int main() {
  if (ll_pose_graph_create(nullptr, 10, 10, nullptr) != LL_ERR_INVALID) return 2;
  if (ll_keyframes_repose(nullptr, nullptr, 0, nullptr, 1, nullptr, nullptr, 0.1f, nullptr, nullptr) != LL_ERR_INVALID) return 2;
  try {
    ll200::Context ctx(0);
    ll200::Pose_graph pg(ctx, 16, 16);
    ll200::MapOfPoses poses;
    ll200::VectorOfConstraints cons;
    for (int i = 0; i < 5; i++) { ll200::Pose3d p; p.p = {{1.0 * i + 0.01 * i * i, 0.02 * i, 0.0}}; poses[i] = p; }
    for (int i = 0; i < 4; i++) { ll200::Constraint3d c; c.id_begin = i; c.id_end = i + 1; c.t_be.p = {{1.0, 0.0, 0.0}}; cons.push_back(c); }
    ll200::Pose3d a = poses[0], b = poses[4];
    cons.push_back(ll200::Pose_graph::add_constrain_of_loop(4, 0, a, b, {{1, 0, 0, 0}}, {{0.0, 0.0, 0.0}}));
    const ll200::MapOfPoses ori = poses;
    const ll_pg_summary s = pg.pose_graph_optimization(poses, cons);
    if (s.iterations < 1 || !(s.final_cost < s.initial_cost) || poses[0].p[0] != 0.0) return 3;
    std::vector<ll200::PointCloud> clouds(5, ll200::PointCloud(10));
    for (auto& c : clouds) for (size_t i = 0; i < c.size(); i++) { c[i].x = 0.5f * i; c[i].y = 1.f; c[i].z = 0.f; c[i].intensity = 3.f; }
    const std::vector<ll200::PointCloud> r = ll200::refine_pointclouds(ctx, clouds, ori, poses, 0.1f);
    if (r.size() != 5 || r[0].size() != 10) return 4;
    std::printf("GPU run: %d iterations, cost %.3g -> %.3g, %zu re-posed points in keyframe 4\n", s.iterations, s.initial_cost, s.final_cost, r[4].size());
  } catch (const ll200::Error& err) {
    if (err.status != LL_ERR_CUDA) { std::printf("unexpected status %d\n", err.status); return 5; }
    std::printf("no GPU: context refused (LL_ERR_CUDA), as it must -- there is no CPU fallback\n");
  }
  return 0;
}
