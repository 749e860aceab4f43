// Compiled, linked against libloamlivox_b200.so and run by tests/test_spin_mapper_cabi.py (no GPU needed to build; without a GPU the run stops
// at the context).  A spinning-lidar odometry node through the C++ mirror: one Laser_feature and one Laser_mapping on one context, a few
// synthetic 16-ring sweeps of a square room, single calls then one sequence call.
#include <cmath>
#include <cstdio>
#include "loamlivox_b200.hpp"

static ll200::PointCloud room_sweep(double x0) {
  ll200::PointCloud in;
  for (int a = 0; a < 1800; a++)
    for (int b = 0; b < 16; b++) {
      const double az = -2 * M_PI * a / 1800, el = (-15.0 + 2.0 * b) * M_PI / 180;
      const double dx = std::cos(el) * std::cos(az), dy = std::cos(el) * std::sin(az), dz = std::sin(el);
      const double wx = dx > 0 ? (5.0 - x0) / dx : (-5.0 - x0) / (dx - 1e-12);
      const double t = std::fmin(std::fmin(wx, 4.0 / std::fabs(dy + 1e-12)), 2.0 / std::fabs(dz + 1e-12));
      ll200::PointXYZI p{}; p.x = (float)(t * dx); p.y = (float)(t * dy); p.z = (float)(t * dz); in.push_back(p);
    }
  return in;
}

int main() {
  if (ll_mapper_process_sweep(nullptr, nullptr, nullptr, 0, LL_FMT_XYZI16, LL_HOST, nullptr, nullptr) != LL_ERR_INVALID) return 2;
  int done = -1;
  if (ll_mapper_process_sweeps(nullptr, nullptr, 1, nullptr, nullptr, LL_FMT_XYZI16, LL_HOST, nullptr, nullptr, &done) != LL_ERR_INVALID || done != 0) return 2;
  try {
    ll200::Context ctx(0);
    ll200::Laser_feature front(ctx, 16);
    ll200::Laser_mapping mapping(ctx);
    ll_reg_result r; ll_mapper_stats st;
    for (int k = 0; k < 3; k++) mapping.process_new_sweep(front, room_sweep(0.02 * k), &r, &st);
    std::vector<ll200::PointCloud> more = {room_sweep(0.06), room_sweep(0.08)};
    std::vector<ll_reg_result> rs;
    mapping.process_new_sweeps(front, more, &rs);
    size_t n = 0;
    front.device_cloud(LL_SPIN_FULL, &n);
    std::printf("GPU run: frame %d, last sweep %d corners %d surfaces, full cloud %zu, t = %.3f\n", mapping.m_current_frame_index, st.n_corner, st.n_surf, n,
                mapping.m_t_w_curr[0]);
    return mapping.m_current_frame_index == 5 && rs.size() == 2 && n == more[1].size() ? 0 : 4;
  } catch (const ll200::Error& err) {
    if (err.status != LL_ERR_CUDA) { std::printf("unexpected status %d\n", err.status); return 6; }
    std::printf("no GPU: context refused (LL_ERR_CUDA), as it must -- there is no CPU fallback\n");
    return 0;
  }
}
