// Prints sizeof / offsetof of ll_loop_closure_cfg and ll_loop_event as "name offset" lines (the struct's size as "sizeof"):
// tests/test_loop_closure_cabi.py compares them with the ctypes mirrors in loam_livox_b200/capi.py.
#include <cstddef>
#include <cstdio>
#include "loamlivox_b200.h"

#define F(T, f) std::printf(#T " " #f " %zu\n", offsetof(T, f))
int main() {
  std::printf("ll_loop_closure_cfg sizeof %zu\n", sizeof(ll_loop_closure_cfg));
  F(ll_loop_closure_cfg, scans_of_each_keyframe); F(ll_loop_closure_cfg, scans_between_two_keyframe); F(ll_loop_closure_cfg, loop); F(ll_loop_closure_cfg, map_alignment_resolution); F(ll_loop_closure_cfg, map_alignment_maximum_icp_iteration);
  F(ll_loop_closure_cfg, map_alignment_inlier_threshold); F(ll_loop_closure_cfg, scene_alignment_maximum_residual_block); F(ll_loop_closure_cfg, surround_pointcloud_resolution); F(ll_loop_closure_cfg, incremental_cov); F(ll_loop_closure_cfg, rng_seed);
  F(ll_loop_closure_cfg, max_cells); F(ll_loop_closure_cfg, reserve_map_points); F(ll_loop_closure_cfg, reserve_history_points); F(ll_loop_closure_cfg, reserve_keyframes);
  std::printf("ll_loop_event sizeof %zu\n", sizeof(ll_loop_event));
  F(ll_loop_event, kind); F(ll_loop_event, keyframe); F(ll_loop_event, ending_frame_idx); F(ll_loop_event, n_candidates); F(ll_loop_event, info);
  F(ll_loop_event, q_wxyz); F(ll_loop_event, t); F(ll_loop_event, his); F(ll_loop_event, scales_run); F(ll_loop_event, decision);
  F(ll_loop_event, status); F(ll_loop_event, inlier_threshold); F(ll_loop_event, icp_q_wxyz); F(ll_loop_event, icp_t); F(ll_loop_event, edge);
  F(ll_loop_event, summary);
  return 0;
}
