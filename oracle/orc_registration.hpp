// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header). PARITY UNPINNED.
// CPU restatement of Point_cloud_registration:
//   loam_livox/source/point_cloud_registration.hpp
//     :163-583 find_out_incremental_transfrom (ICP outer loop, gates, cap drop, 2 solves, inlier select, reject)
//     :585-605 4-argument overload (builds the trees itself)
//     :622-661 pointAssociateToMap (+ :607-620 compute_interpolatation_rodrigue, :128-141 refine_blur)
//     :153-161 compute_inlier_residual_threshold
//   state hand-off  loam_livox/source/laser_mapping.hpp:1266-1297 init_pointcloud_registration
// Residual-block cap (:232-238,:339-345,:434-458): the reference draws from a std::random_device-seeded mt19937
// (include/tools/tools_random.hpp:18-25), which no second implementation can reproduce.  The RULE is restated exactly
// (pre-skip of a feature when rand*N > 2*cap with N the feature count of its class; after the block list is built, when its size M exceeds
// the cap, block i is dropped when rand_i > (float)cap/(float)M), and the random numbers come from a counter-based generator
// cap_uniform(seed, icp_iteration, stream, index) with a caller-supplied seed (RegParams::rng_seed), so that the CUDA path can draw the
// very same numbers: stream 0 / 1 = corner / surface pre-skip (index = feature index), stream 2 = drop (index = slot of the block =
// feature index, surfaces offset by the corner count; the reference indexes its array by list position, an i.i.d. relabelling).
#pragma once
#include <set>
#include <vector>
#include "orc_cloud.hpp"
#include "orc_solver.hpp"

namespace orc {

struct RegParams {  // fields init_pointcloud_registration copies + the members scene_alignment pokes
  int if_motion_deblur = 0;
  int current_frame_index = 1000, mapping_init_accumulate_frames = 50;
  float para_max_angular_rate = 200.0f / 50.0f, para_max_speed = 100.0f / 50.0f, max_final_cost = 100.0f;
  int icp_max_iterations = 20, cere_max_iterations = 100, cere_prerun_times = 2;
  float minimum_pt_time_stamp = 0.f, maximum_pt_time_stamp = 1.0f;
  double minimum_icp_R_diff = 0.01, minimum_icp_T_diff = 0.01;
  double inliner_dis = 0.02, inlier_ratio = 0.80;
  double maximum_dis_plane_for_match = 50.0, maximum_dis_line_for_match = 2.0;
  int icp_plane = 1, icp_line = 1;
  int maximum_allow_residual_block = 100000;
  double huber_a = 0.1;
  double q_w_last[4] = {1, 0, 0, 0};  // w,x,y,z
  double t_w_last[3] = {0, 0, 0};
  double q_w_curr[4] = {1, 0, 0, 0};
  double t_w_curr[3] = {0, 0, 0};
  double para_buffer_incremental[7] = {0, 0, 0, 1, 0, 0, 0};  // q (x,y,z,w), t
  int num_threads = 1;  // CPU-baseline knob (reference is single-threaded)
  int rng_seed = 0;     // seed of the counter-based generator that stands in for m_rand_float (see the header comment)
};

// Counter-based uniform float in [0,1): splitmix64 finaliser over (seed, ICP iteration, stream, index), top 24 bits.
inline float cap_uniform(int seed, int icp_iter, int stream, int index) {
  unsigned long long z = (unsigned long long)(unsigned)seed * 0x9E3779B97F4A7C15ull + (((unsigned long long)(unsigned)icp_iter << 40) | ((unsigned long long)(unsigned)stream << 32) | (unsigned long long)(unsigned)index);
  z ^= z >> 30; z *= 0xbf58476d1ce4e5b9ull; z ^= z >> 27; z *= 0x94d049bb133111ebull; z ^= z >> 31;
  return (float)(z >> 40) * (1.0f / 16777216.0f);
}

struct RegResult {
  int status = 1;  // return value of find_out_incremental_transfrom: 1 accepted-or-skipped, 0 rejected
  int registered = 0;  // 1 if the ICP branch actually ran (:199)
  double q_w_curr[4], t_w_curr[3];
  double q_w_incre[4], t_w_incre[3];  // q as w,x,y,z
  double inlier_threshold = 0, final_cost = 0, initial_cost = 0;
  int num_residual_blocks = 0, icp_iterations = 0, corner_used = 0, surf_used = 0;
  double angular_diff = 0, t_diff = 0;
  int total_lm_iterations = 0, total_cost_evals = 0, total_jac_evals = 0, total_line_search_steps = 0;
};

struct IcpIterTrace {  // per ICP iteration, for step-by-step parity tests
  int corner_avail, surf_avail, blocks_before_select, blocks_after_select;
  double inlier_threshold; double x_after_solve1[7]; double x_after_solve2[7];
  double cost1_initial, cost1_final, cost2_initial, cost2_final; int lm_iters1, lm_iters2;
};

struct Registration {
  RegParams P;
  Qd q_w_last, q_w_curr; V3d t_w_last, t_w_curr;
  double buf[7];  // m_para_buffer_incremental
  double interp_theta = 0; double omega_hat[3][3] = {}, omega_hat_sq2[3][3] = {};
  double inlier_threshold = 0;
  std::vector<IcpIterTrace> trace;

  void init(const RegParams& p) {
    P = p;
    q_w_last = {p.q_w_last[0], p.q_w_last[1], p.q_w_last[2], p.q_w_last[3]}; t_w_last = {p.t_w_last[0], p.t_w_last[1], p.t_w_last[2]};
    q_w_curr = {p.q_w_curr[0], p.q_w_curr[1], p.q_w_curr[2], p.q_w_curr[3]}; t_w_curr = {p.t_w_curr[0], p.t_w_curr[1], p.t_w_curr[2]};
    for (int k = 0; k < 7; k++) buf[k] = p.para_buffer_incremental[k];
  }

  float refine_blur(float in_blur, float min_blur, float max_blur) const {  // :128-141
    float res = 1.0f;
    if (P.if_motion_deblur) { res = (in_blur - min_blur) / (max_blur - min_blur); if (!std::isfinite(res) || res > 1.0) return 1.0f; else return res; }
    return res;
  }

  void compute_interpolatation_rodrigue() {  // :607-620, Eigen::AngleAxisd(q)
    Qd q{buf[3], buf[0], buf[1], buf[2]};
    double n = std::sqrt(q.x * q.x + q.y * q.y + q.z * q.z);
    double axis[3]; double angle;
    if (n != 0.0) { angle = 2.0 * std::atan2(n, std::fabs(q.w)); if (q.w < 0) n = -n; axis[0] = q.x / n; axis[1] = q.y / n; axis[2] = q.z / n; }
    else { angle = 0; axis[0] = 1; axis[1] = 0; axis[2] = 0; }
    double an = std::sqrt(axis[0] * axis[0] + axis[1] * axis[1] + axis[2] * axis[2]);
    for (int k = 0; k < 3; k++) axis[k] /= an;
    interp_theta = angle;
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) omega_hat[i][j] = 0;
    omega_hat[0][1] = -axis[2]; omega_hat[1][0] = axis[2]; omega_hat[0][2] = axis[1]; omega_hat[2][0] = -axis[1]; omega_hat[1][2] = -axis[0]; omega_hat[2][1] = axis[0];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) { double s = 0; for (int k = 0; k < 3; k++) s += omega_hat[i][k] * omega_hat[k][j]; omega_hat_sq2[i][j] = s; }
  }

  // :622-661. pi/po: 4 floats (x,y,z,intensity)
  void pointAssociateToMap(const float* pi, float* po, double interpolate_s = 1.0, int if_undistore = 0) const {
    V3d pc{pi[0], pi[1], pi[2]}; V3d pw;
    if (P.if_motion_deblur == 0 || if_undistore == 0 || interpolate_s == 1.0) pw = qrot(q_w_curr, pc) + t_w_curr;
    else {
      V3d iT{buf[4] * (interpolate_s * 1.0), buf[5] * (interpolate_s * 1.0), buf[6] * (interpolate_s * 1.0)};
      double th = interp_theta * interpolate_s; double R[3][3];
      for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) R[i][j] = (i == j ? 1.0 : 0.0) + std::sin(th) * omega_hat[i][j] + (1 - std::cos(th)) * omega_hat_sq2[i][j];
      V3d rp{R[0][0] * pc.x + R[0][1] * pc.y + R[0][2] * pc.z, R[1][0] * pc.x + R[1][1] * pc.y + R[1][2] * pc.z, R[2][0] * pc.x + R[2][1] * pc.y + R[2][2] * pc.z};
      pw = qrot(q_w_last, rp + iT) + t_w_last;
    }
    po[0] = (float)pw.x; po[1] = (float)pw.y; po[2] = (float)pw.z; po[3] = pi[3];
  }

  static double inlier_residual_threshold(const std::vector<double>& residuals, double ratio) {  // :153-161
    std::set<double> dis_vec;
    for (size_t i = 0; i < residuals.size() / 3; i++) dis_vec.insert(std::fabs(residuals[3 * i + 0]) + std::fabs(residuals[3 * i + 1]) + std::fabs(residuals[3 * i + 2]));
    return *(std::next(dis_vec.begin(), (int)(ratio * dis_vec.size())));
  }

  // Builds the residual blocks of one ICP iteration (:230-432). knn_*: precomputed trees.
  void build_blocks(const float* map_c, const KdTree& tree_c, const float* map_s, const KdTree& tree_s,
                    const float* scan_c, int nc, const float* scan_s, int ns, std::vector<ResidualBlock>& blocks, int* corner_avail, int* surf_avail, int icp_iter = 0) const {
    const int K = 5; const int if_undistore_in_matching = 1;
    std::vector<int> c_idx((size_t)nc * K, -1), s_idx((size_t)ns * K, -1); std::vector<float> c_d((size_t)nc * K, 0.f), s_d((size_t)ns * K, 0.f);
    std::vector<int> c_found(nc, 0), s_found(ns, 0);
    std::vector<float> c_sel((size_t)nc * 4), s_sel((size_t)ns * 4);
#pragma omp parallel for num_threads(P.num_threads) schedule(dynamic, 256) if (P.num_threads > 1)
    for (int i = 0; i < nc; i++) {
      const float* po = scan_c + (size_t)i * 4;
      if (nc > 2 * P.maximum_allow_residual_block && cap_uniform(P.rng_seed, icp_iter, 0, i) * nc > 2 * P.maximum_allow_residual_block) { c_found[i] = -1; continue; }  // :232-238
      if (!std::isfinite(po[0]) || !std::isfinite(po[1]) || !std::isfinite(po[2])) { c_found[i] = -1; continue; }
      pointAssociateToMap(po, &c_sel[(size_t)i * 4], refine_blur(po[3], P.minimum_pt_time_stamp, P.maximum_pt_time_stamp), if_undistore_in_matching);
      c_found[i] = tree_c.knn(&c_sel[(size_t)i * 4], K, &c_idx[(size_t)i * K], &c_d[(size_t)i * K]);
    }
#pragma omp parallel for num_threads(P.num_threads) schedule(dynamic, 256) if (P.num_threads > 1)
    for (int i = 0; i < ns; i++) {
      const float* po = scan_s + (size_t)i * 4;
      if (ns > 2 * P.maximum_allow_residual_block && cap_uniform(P.rng_seed, icp_iter, 1, i) * ns > 2 * P.maximum_allow_residual_block) { s_found[i] = -1; continue; }  // :339-345
      pointAssociateToMap(po, &s_sel[(size_t)i * 4], refine_blur(po[3], P.minimum_pt_time_stamp, P.maximum_pt_time_stamp), if_undistore_in_matching);
      s_found[i] = tree_s.knn(&s_sel[(size_t)i * 4], K, &s_idx[(size_t)i * K], &s_d[(size_t)i * K]);
    }
    *corner_avail = 0; *surf_avail = 0;
    for (int i = 0; i < nc; i++) {
      if (c_found[i] != K) continue;  // :242-252
      if (c_d[(size_t)i * K + K - 1] < P.maximum_dis_line_for_match) {
        if (P.icp_line) {
          const float* po = scan_c + (size_t)i * 4; double cp[3] = {po[0], po[1], po[2]};
          const float* m1 = map_c + (size_t)c_idx[(size_t)i * K + 0] * 4; const float* m2 = map_c + (size_t)c_idx[(size_t)i * K + 1] * 4;
          double p1[3] = {m1[0], m1[1], m1[2]}, p2[3] = {m2[0], m2[1], m2[2]};
          double dn = std::sqrt((p1[0] - p2[0]) * (p1[0] - p2[0]) + (p1[1] - p2[1]) * (p1[1] - p2[1]) + (p1[2] - p2[2]) * (p1[2] - p2[2]));
          if (dn < 0.0001) continue;  // :302-303
          ResidualBlock b; make_point2line(b, cp, p1, p2);
          if (P.if_motion_deblur) { b.motion_blur = 1; b.s = refine_blur(po[3], P.minimum_pt_time_stamp, P.maximum_pt_time_stamp) * 1.0; }
          b.src = 0; b.src_index = i; blocks.push_back(b); (*corner_avail)++;
        }
      }
    }
    for (int i = 0; i < ns; i++) {
      // :351-353 — the reference neither checks the point nor the kNN return count here; with fewer than 5
      // neighbours (map smaller than 5 points) it would read stale data. SURFACE_MIN_MAP_NUM = 50 rules that out.
      if (s_found[i] != K) continue;
      if (s_d[(size_t)i * K + K - 1] < P.maximum_dis_plane_for_match) {
        if (P.icp_plane) {
          const float* po = scan_s + (size_t)i * 4; double cp[3] = {po[0], po[1], po[2]};
          const float* m0 = map_s + (size_t)s_idx[(size_t)i * K + 0] * 4; const float* m1 = map_s + (size_t)s_idx[(size_t)i * K + K / 2] * 4; const float* m2 = map_s + (size_t)s_idx[(size_t)i * K + K - 1] * 4;
          double a[3] = {m0[0], m0[1], m0[2]}, b3[3] = {m1[0], m1[1], m1[2]}, c3[3] = {m2[0], m2[1], m2[2]};
          ResidualBlock b; make_point2plane(b, cp, a, b3, c3);
          if (P.if_motion_deblur) { b.motion_blur = 1; b.s = refine_blur(po[3], P.minimum_pt_time_stamp, P.maximum_pt_time_stamp) * 1.0; }
          b.src = 1; b.src_index = i; blocks.push_back(b);
        }
        (*surf_avail)++;
      }
    }
  }

  // :163-583
  int find_out_incremental_transfrom(const float* map_c, int nmc, const KdTree& tree_c, const float* map_s, int nms, const KdTree& tree_s,
                                     const float* scan_c, int nc, const float* scan_s, int ns, RegResult* out) {
    RegResult R; trace.clear();
    int corner_avail = 0, surf_avail = 0; float minimize_cost = 0; SolveSummary summary;
    double angular_diff = 0, t_diff = 0; int iterCount = 0;
    if (nmc > 0 && nms > 50 && P.current_frame_index > P.mapping_init_accumulate_frames) {
      R.registered = 1;
      Qd q_last_optimize{1, 0, 0, 0}; V3d t_last_optimize{0, 0, 0};
      for (iterCount = 0; iterCount < P.icp_max_iterations; iterCount++) {
        Problem prob; prob.q_last = q_w_last; prob.t_last = t_w_last; prob.huber_a = P.huber_a; prob.t_bound = P.para_max_speed; prob.num_threads = P.num_threads;
        build_blocks(map_c, tree_c, map_s, tree_s, scan_c, nc, scan_s, ns, prob.blocks, &corner_avail, &surf_avail, iterCount);
        if (prob.blocks.size() > (size_t)P.maximum_allow_residual_block) {  // :434-458 drop some of the residual blocks
          const float threshold_to_reserve = (float)P.maximum_allow_residual_block / (float)prob.blocks.size();
          std::vector<ResidualBlock> kept0; kept0.reserve(prob.blocks.size());
          for (const ResidualBlock& b : prob.blocks)
            if (!(cap_uniform(P.rng_seed, iterCount, 2, b.src == 0 ? b.src_index : nc + b.src_index) > threshold_to_reserve)) kept0.push_back(b);
          prob.blocks.swap(kept0);
        }
        IcpIterTrace tr{}; tr.corner_avail = corner_avail; tr.surf_avail = surf_avail; tr.blocks_before_select = (int)prob.blocks.size();
        if (prob.blocks.empty()) { out->status = -3; return -3; }  // reference would dereference an empty std::set (:160)
        SolveOptions so; so.max_num_iterations = P.cere_prerun_times;  // :466-467
        solve(prob, so, buf, &summary);
        R.total_lm_iterations += summary.iterations; R.total_cost_evals += summary.num_cost_evals; R.total_jac_evals += summary.num_jac_evals; R.total_line_search_steps += summary.num_line_search_steps;
        tr.cost1_initial = summary.initial_cost; tr.cost1_final = summary.final_cost; tr.lm_iters1 = summary.iterations; for (int k = 0; k < 7; k++) tr.x_after_solve1[k] = buf[k];
        // :476-499 Evaluate (loss applied) -> threshold -> drop outliers
        double total_cost = 0; std::vector<double> residuals;
        prob.evaluate(buf, &total_cost, &residuals, nullptr, nullptr); R.total_cost_evals++;
        double ratio_thr = inlier_residual_threshold(residuals, P.inlier_ratio);
        inlier_threshold = std::max(P.inliner_dis, ratio_thr);
        std::vector<ResidualBlock> kept; kept.reserve(prob.blocks.size());
        for (size_t i = 0; i < prob.blocks.size(); i++)
          if (!((std::fabs(residuals[3 * i + 0]) + std::fabs(residuals[3 * i + 1]) + std::fabs(residuals[3 * i + 2])) > inlier_threshold)) kept.push_back(prob.blocks[i]);
        prob.blocks.swap(kept);
        tr.blocks_after_select = (int)prob.blocks.size(); tr.inlier_threshold = inlier_threshold;
        so.max_num_iterations = P.cere_max_iterations;  // :501-508
        solve(prob, so, buf, &summary);
        R.total_lm_iterations += summary.iterations; R.total_cost_evals += summary.num_cost_evals; R.total_jac_evals += summary.num_jac_evals; R.total_line_search_steps += summary.num_line_search_steps;
        tr.cost2_initial = summary.initial_cost; tr.cost2_final = summary.final_cost; tr.lm_iters2 = summary.iterations; for (int k = 0; k < 7; k++) tr.x_after_solve2[k] = buf[k];
        trace.push_back(tr);
        if (P.if_motion_deblur) compute_interpolatation_rodrigue();  // :509-513
        Qd q_incre{buf[3], buf[0], buf[1], buf[2]}; V3d t_incre{buf[4], buf[5], buf[6]};
        t_w_curr = qrot(q_w_last, t_incre) + t_w_last;  // :514-515
        q_w_curr = qmul(q_w_last, q_incre);
        angular_diff = (float)angular_distance(q_w_curr, q_w_last) * 57.3;  // :517
        t_diff = norm(t_w_curr - t_w_last);
        minimize_cost = (float)summary.final_cost;
        if (angular_distance(q_last_optimize, q_incre) < 57.3 * P.minimum_icp_R_diff && norm(t_last_optimize - t_incre) < P.minimum_icp_T_diff) break;  // :521-526
        q_last_optimize = q_incre; t_last_optimize = t_incre;
      }
      inlier_threshold = inlier_threshold * summary.final_cost / summary.initial_cost;  // :559
      R.icp_iterations = std::min(iterCount + 1, P.icp_max_iterations);
      if (angular_diff > P.para_max_angular_rate || minimize_cost > P.max_final_cost) {  // :561-573
        q_w_curr = q_w_last; t_w_curr = t_w_last; R.status = 0;
      }
    }
    R.q_w_curr[0] = q_w_curr.w; R.q_w_curr[1] = q_w_curr.x; R.q_w_curr[2] = q_w_curr.y; R.q_w_curr[3] = q_w_curr.z;
    R.t_w_curr[0] = t_w_curr.x; R.t_w_curr[1] = t_w_curr.y; R.t_w_curr[2] = t_w_curr.z;
    R.q_w_incre[0] = buf[3]; R.q_w_incre[1] = buf[0]; R.q_w_incre[2] = buf[1]; R.q_w_incre[3] = buf[2];
    R.t_w_incre[0] = buf[4]; R.t_w_incre[1] = buf[5]; R.t_w_incre[2] = buf[6];
    R.inlier_threshold = inlier_threshold; R.final_cost = summary.final_cost; R.initial_cost = summary.initial_cost; R.num_residual_blocks = summary.num_residual_blocks;
    R.corner_used = corner_avail; R.surf_used = surf_avail; R.angular_diff = angular_diff; R.t_diff = t_diff;
    *out = R; return R.status;
  }
};

}  // namespace orc
