// Compiled, linked against libloamlivox_b200.so and run by tests/test_recovery_cabi.py (no GPU needed to build; without a GPU the run stops at
// the context).  The recovery calls of the C API and Laser_mapping::set_recovery / recovery_log of the C++ mirror on a few tiny scans.
#include <cstdio>
#include "loamlivox_b200.hpp"

int main() {
  ll_recovery_cfg cfg; ll_mapper_recovery_default(&cfg);
  ll_recovery_step e[1]; int n = -1, dropped = -1; size_t cnt[4];
  if (ll_mapper_set_recovery(nullptr, &cfg) != LL_ERR_INVALID || ll_mapper_set_recovery(nullptr, nullptr) != LL_ERR_INVALID) return 2;
  if (ll_mapper_recovery_read(nullptr, e, 1, &n, &dropped) != LL_ERR_INVALID) return 2;
  if (ll_mapper_recovery_last_inputs(nullptr, nullptr, nullptr, nullptr, cnt, nullptr, nullptr, nullptr, nullptr, 0, nullptr, nullptr, 0) != LL_ERR_INVALID) return 2;
  try {
    ll200::Context ctx(0);
    ll200::Laser_mapping mapping(ctx);
    mapping.set_recovery(&cfg);
    ll200::PointCloud raw(200);
    for (size_t i = 0; i < raw.size(); i++) { raw[i].x = 5.f; raw[i].y = 0.01f * i; raw[i].z = 0.f; raw[i].intensity = 10.f; }
    mapping.process_new_scans({raw, raw}, {100.0, 100.1});
    int d = 0;
    const std::vector<ll_recovery_step> log = mapping.recovery_log(&d);
    mapping.set_recovery(nullptr);
    std::printf("GPU run: %zu log entries, %d dropped\n", log.size(), d);
  } catch (const ll200::Error& err) {
    if (err.status != LL_ERR_CUDA) { std::printf("unexpected status %d\n", err.status); return 5; }
    std::printf("no GPU: context refused (LL_ERR_CUDA), as it must -- there is no CPU fallback\n");
  }
  return 0;
}
