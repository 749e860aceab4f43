// Compiled, linked against libloamlivox_b200.so and run by tests/test_spin_cabi.py (no GPU needed to build; without a GPU the run stops at the
// context).  Laser_feature's Velodyne branch through the C++ mirror: one synthetic 16-ring sweep of a square room.
#include <cmath>
#include <cstdio>
#include "loamlivox_b200.hpp"

int main() {
  ll_spin_cfg cfg; ll_spin_cfg_default(&cfg);
  if (cfg.scan_line != 16 || cfg.max_points != 400000 || std::fabs(cfg.minimum_range - 0.1f) > 0 || std::fabs(cfg.plane_resolution - 0.4f) > 0) return 2;
  if (ll_spin_create(nullptr, &cfg, nullptr) != LL_ERR_INVALID) return 2;
  if (ll_spin_extract(nullptr, nullptr, 0, LL_FMT_XYZI16, LL_HOST, nullptr) != LL_ERR_INVALID) return 2;
  try {
    ll200::Context ctx(0);
    ll200::Laser_feature lf(ctx, 16);
    ll200::PointCloud in;
    for (int a = 0; a < 1800; a++)
      for (int b = 0; b < 16; b++) {
        const double az = -2 * M_PI * a / 1800, el = (-15.0 + 2.0 * b) * M_PI / 180;
        const double dx = std::cos(el) * std::cos(az), dy = std::cos(el) * std::sin(az), dz = std::sin(el);
        const double t = std::fmin(std::fmin(5.0 / std::fabs(dx + 1e-12), 4.0 / std::fabs(dy + 1e-12)), 2.0 / std::fabs(dz + 1e-12));
        ll200::PointXYZI p{}; p.x = (float)(t * dx); p.y = (float)(t * dy); p.z = (float)(t * dz); in.push_back(p);
      }
    lf.laserCloudHandler(in);
    size_t n = 0;
    if (!lf.device_cloud(LL_SPIN_LESS_FLAT, &n) || n != lf.surfPointsLessFlat.size()) return 3;
    std::printf("GPU run: full %zu sharp %zu less sharp %zu flat %zu less flat %zu\n", lf.laserCloud.size(), lf.cornerPointsSharp.size(), lf.cornerPointsLessSharp.size(),
                lf.surfPointsFlat.size(), lf.surfPointsLessFlat.size());
    return lf.laserCloud.size() == in.size() && !lf.surfPointsFlat.empty() ? 0 : 4;
  } catch (const ll200::Error& err) {
    if (err.status != LL_ERR_CUDA) { std::printf("unexpected status %d\n", err.status); return 6; }
    std::printf("no GPU: context refused (LL_ERR_CUDA), as it must -- there is no CPU fallback\n");
    return 0;
  }
}
