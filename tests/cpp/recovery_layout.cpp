// Prints sizeof / offsetof of ll_recovery_cfg and ll_recovery_step as "name offset" lines (the struct's size as "sizeof"): tests/test_recovery_cabi.py
// compares them with the ctypes mirrors in loam_livox_b200/capi.py.
#include <cstddef>
#include <cstdio>
#include "loamlivox_b200.h"

#define F(T, f) std::printf(#T " " #f " %zu\n", offsetof(T, f))
int main() {
  std::printf("ll_recovery_cfg sizeof %zu\n", sizeof(ll_recovery_cfg));
  F(ll_recovery_cfg, max_inlier_threshold); F(ll_recovery_cfg, lost_after); F(ll_recovery_cfg, trunc); F(ll_recovery_cfg, res); F(ll_recovery_cfg, score_leaf);
  F(ll_recovery_cfg, yaw_step_deg); F(ll_recovery_cfg, t_step); F(ll_recovery_cfg, window_base); F(ll_recovery_cfg, window_growth);
  F(ll_recovery_cfg, max_candidates); F(ll_recovery_cfg, max_hypotheses); F(ll_recovery_cfg, fine_yaw_step_deg); F(ll_recovery_cfg, fine_t_step);
  F(ll_recovery_cfg, fine_t_half); F(ll_recovery_cfg, min_verify_fraction); F(ll_recovery_cfg, reserve_field_voxels); F(ll_recovery_cfg, reserve_whole_map_points);
  std::printf("ll_recovery_step sizeof %zu\n", sizeof(ll_recovery_step));
  F(ll_recovery_step, frame_index); F(ll_recovery_step, state_before); F(ll_recovery_step, state_after); F(ll_recovery_step, bad); F(ll_recovery_step, bad_steps);
  F(ll_recovery_step, appended); F(ll_recovery_step, attempted); F(ll_recovery_step, attempt_status); F(ll_recovery_step, nt); F(ll_recovery_step, n_yaw);
  F(ll_recovery_step, n_cand); F(ll_recovery_step, best); F(ll_recovery_step, adopted); F(ll_recovery_step, grew); F(ll_recovery_step, n_score);
  F(ll_recovery_step, score_leaf); F(ll_recovery_step, t0); F(ll_recovery_step, step); F(ll_recovery_step, tilt_wxyz); F(ll_recovery_step, verify_fraction);
  F(ll_recovery_step, q_wxyz); F(ll_recovery_step, t); F(ll_recovery_step, inlier_threshold); F(ll_recovery_step, ms_map); F(ll_recovery_step, ms_search);
  return 0;
}
