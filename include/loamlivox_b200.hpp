// loamlivox_b200.hpp — header-only C++ mirror of the reference's classes for the hot path, over the C-ABI (loamlivox_b200.h).
// Same names, argument meaning and return conventions as
//   Livox_laser                      loam_livox/source/livox_feature_extractor.hpp:77   (extract_laser_features :722, get_features :219)
//   Point_cloud_registration         loam_livox/source/point_cloud_registration.hpp:38  (find_out_incremental_transfrom :163/:585,
//                                                                                               pointcloudAssociateToMap :673)
//   Points_cloud_map                 loam_livox/source/cell_map_keyframe.hpp:264        (append_cloud :619, cells in radius + FOV :761, laser_mapping.hpp:475-516)
//   Laser_mapping::process_new_scan  loam_livox/source/laser_mapping.hpp:1316
// so that laser_feature_extractor.hpp / laser_mapping.hpp can switch with the small adapter shown in INTEGRATION.md.
// No PCL / Eigen / Ceres needed: clouds are std::vector<ll200::PointXYZI> (layout-identical to pcl::PointXYZI, 32 bytes).
#pragma once
#include <array>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>
#include "loamlivox_b200.h"

namespace ll200 {

struct alignas(16) PointXYZI { float x, y, z, _pad0; float intensity, _pad1, _pad2, _pad3; };   // == pcl::PointXYZI
static_assert(sizeof(PointXYZI) == sizeof(ll_pcl_xyzi), "layout");
typedef std::vector<PointXYZI> PointCloud;

struct Error : std::runtime_error { int status; Error(int s, const std::string& m) : std::runtime_error(m), status(s) {} };

class Context {
 public:
  explicit Context(int device = 0, const ll_config* cfg = nullptr) {
    int st = ll_ctx_create(cfg, device, &ctx_);
    if (st != LL_OK) throw Error(st, "ll_ctx_create failed: a CUDA device (sm_90a) is required, there is no CPU fallback");
  }
  ~Context() { ll_ctx_destroy(ctx_); }
  Context(const Context&) = delete; Context& operator=(const Context&) = delete;
  ll_ctx* get() const { return ctx_; }
  void check(int st) const { if (st != LL_OK) throw Error(st, ll_last_error(ctx_)); }
  void warmup() { check(ll_ctx_warmup(ctx_)); }   // first-use costs (module loads, first cooperative launch) now instead of in the first registration
 private:
  ll_ctx* ctx_ = nullptr;
};

inline PointCloud to_cloud(const std::vector<ll_point>& p) {
  PointCloud c(p.size());
  for (size_t i = 0; i < p.size(); i++) { c[i].x = p[i].x; c[i].y = p[i].y; c[i].z = p[i].z; c[i]._pad0 = 1.f; c[i].intensity = p[i].intensity; c[i]._pad1 = c[i]._pad2 = c[i]._pad3 = 0.f; }
  return c;
}

// ---- Livox_laser ------------------------------------------------------------------------------------------
class Livox_laser {
 public:
  explicit Livox_laser(Context& ctx) : ctx_(ctx) { ctx_.check(ll_extract_reset(ctx_.get())); }
  // returns laserCloudScans.size(): the number of rosette petals handed back (the caller drops the frame when <= 5)
  int extract_laser_features(const PointCloud& laserCloudIn, double time_stamp) {
    int n_scans = 0; n_ = laserCloudIn.size();
    ctx_.check(ll_extract(ctx_.get(), laserCloudIn.data(), n_, LL_FMT_PCL32, LL_HOST, time_stamp, &n_scans));
    return n_scans;
  }
  void get_features(PointCloud& pc_corners, PointCloud& pc_surface, PointCloud& pc_full_res, float minimum_blur = 0.0f, float maximum_blur = 0.3f) {
    std::vector<ll_point> c(n_), s(n_), f(n_); size_t nc = 0, ns = 0, nf = 0;
    ctx_.check(ll_get_features(ctx_.get(), minimum_blur, maximum_blur, c.data(), &nc, s.data(), &ns, f.data(), &nf));
    c.resize(nc); s.resize(ns); f.resize(nf);
    pc_corners = to_cloud(c); pc_surface = to_cloud(s); pc_full_res = to_cloud(f);
  }
  void piece_bounds(int pieces, std::vector<float>& start, std::vector<float>& end) {
    start.resize(pieces); end.resize(pieces); ctx_.check(ll_piece_bounds(ctx_.get(), pieces, start.data(), end.data()));
  }
 private:
  Context& ctx_; size_t n_ = 0;
};

// ---- pcl::VoxelGrid<PointXYZI>::filter --------------------------------------------------------------------
inline PointCloud voxel_grid_filter(Context& ctx, const PointCloud& in, float leaf) {
  std::vector<ll_point> out(in.size()); size_t m = 0;
  ctx.check(ll_voxel_downsample(ctx.get(), in.data(), in.size(), LL_FMT_PCL32, LL_HOST, leaf, out.data(), &m));
  out.resize(m); return to_cloud(out);
}

// ---- the pair of KdTreeFLANN snapshots of update_buff_for_matching (laser_mapping.hpp:533-559) --------------
class Match_map {
 public:
  Match_map(Context& ctx, const PointCloud& corner_from_map, const PointCloud& surf_from_map) : ctx_(ctx) {
    ctx_.check(ll_map_build(ctx_.get(), corner_from_map.data(), corner_from_map.size(), surf_from_map.data(), surf_from_map.size(), LL_FMT_PCL32, LL_HOST, &map_));
  }
  ~Match_map() { ll_map_release(map_); }
  Match_map(const Match_map&) = delete; Match_map& operator=(const Match_map&) = delete;
  const ll_map* get() const { return map_; }
 private:
  Context& ctx_; ll_map* map_ = nullptr;
};

// ---- Point_cloud_registration -----------------------------------------------------------------------------
class Point_cloud_registration {
 public:
  // the public members Laser_mapping::init_pointcloud_registration writes (laser_mapping.hpp:1266-1297); quaternions (w,x,y,z)
  int m_if_motion_deblur = 0, m_current_frame_index = 0, m_mapping_init_accumulate_frames = 100;
  float m_para_max_angular_rate = 200.0f / 50.0f, m_para_max_speed = 100.0f / 50.0f, m_max_final_cost = 100.0f;
  int m_para_icp_max_iterations = 20, m_para_cere_max_iterations = 100, m_para_cere_prerun_times = 2;
  float m_minimum_pt_time_stamp = 0, m_maximum_pt_time_stamp = 1.0f;
  double m_minimum_icp_R_diff = 0.01, m_minimum_icp_T_diff = 0.01, m_inliner_dis = 0.02, m_inlier_ratio = 0.80;
  double m_maximum_dis_plane_for_match = 50.0, m_maximum_dis_line_for_match = 2.0;
  int ICP_PLANE = 1, ICP_LINE = 1, m_maximum_allow_residual_block = 100000;
  int m_rand_seed = 0;   // stands in for m_rand_float's std::random_device seed (tools_random.hpp:18-25): same seed, same dropped residual blocks
  std::array<double, 4> m_q_w_last{{1, 0, 0, 0}}, m_q_w_curr{{1, 0, 0, 0}}, m_q_w_incre{{1, 0, 0, 0}};
  std::array<double, 3> m_t_w_last{{0, 0, 0}}, m_t_w_curr{{0, 0, 0}}, m_t_w_incre{{0, 0, 0}};
  double m_inlier_threshold = 0;
  ll_reg_result m_final_opt_summary{};   // final_cost / num_residual_blocks etc. (ceres::Solver::Summary stand-in)

  explicit Point_cloud_registration(Context& ctx) : ctx_(ctx) {}

  // 1 = accepted or skipped, 0 = rejected (pose reverted) — point_cloud_registration.hpp:572,581
  int find_out_incremental_transfrom(const Match_map& map, const PointCloud& laserCloudCornerStack, const PointCloud& laserCloudSurfStack) {
    ll_reg_state s; ll_reg_state_default(&s);
    s.if_motion_deblur = m_if_motion_deblur; s.current_frame_index = m_current_frame_index; s.mapping_init_accumulate_frames = m_mapping_init_accumulate_frames;
    s.icp_max_iterations = m_para_icp_max_iterations; s.cere_max_iterations = m_para_cere_max_iterations; s.cere_prerun_times = m_para_cere_prerun_times;
    s.icp_plane = ICP_PLANE; s.icp_line = ICP_LINE; s.maximum_allow_residual_block = m_maximum_allow_residual_block; s.rng_seed = m_rand_seed;
    s.para_max_angular_rate = m_para_max_angular_rate; s.para_max_speed = m_para_max_speed; s.max_final_cost = m_max_final_cost;
    s.minimum_pt_time_stamp = m_minimum_pt_time_stamp; s.maximum_pt_time_stamp = m_maximum_pt_time_stamp;
    s.minimum_icp_R_diff = m_minimum_icp_R_diff; s.minimum_icp_T_diff = m_minimum_icp_T_diff; s.inliner_dis = m_inliner_dis; s.inlier_ratio = m_inlier_ratio;
    s.maximum_dis_plane_for_match = m_maximum_dis_plane_for_match; s.maximum_dis_line_for_match = m_maximum_dis_line_for_match;
    for (int k = 0; k < 4; k++) { s.q_w_last[k] = m_q_w_last[k]; s.q_w_curr[k] = m_q_w_curr[k]; }
    for (int k = 0; k < 3; k++) { s.t_w_last[k] = m_t_w_last[k]; s.t_w_curr[k] = m_t_w_curr[k]; }
    s.para_buffer_incremental[0] = m_q_w_incre[1]; s.para_buffer_incremental[1] = m_q_w_incre[2]; s.para_buffer_incremental[2] = m_q_w_incre[3]; s.para_buffer_incremental[3] = m_q_w_incre[0];
    for (int k = 0; k < 3; k++) s.para_buffer_incremental[4 + k] = m_t_w_incre[k];
    ll_reg_result r;
    ctx_.check(ll_register(ctx_.get(), map.get(), laserCloudCornerStack.data(), laserCloudCornerStack.size(), laserCloudSurfStack.data(), laserCloudSurfStack.size(),
                           LL_FMT_PCL32, LL_HOST, &s, &r));
    for (int k = 0; k < 4; k++) { m_q_w_curr[k] = r.q_w_curr[k]; m_q_w_incre[k] = r.q_w_incre[k]; }
    for (int k = 0; k < 3; k++) { m_t_w_curr[k] = r.t_w_curr[k]; m_t_w_incre[k] = r.t_w_incre[k]; }
    m_inlier_threshold = r.inlier_threshold; m_final_opt_summary = r;
    return r.status;
  }
  // pointcloudAssociateToMap (:673-685), non-deblur branch
  unsigned int pointcloudAssociateToMap(const PointCloud& pc_in, PointCloud& pt_out) {
    std::vector<ll_point> out(pc_in.size());
    ctx_.check(ll_transform(ctx_.get(), m_q_w_curr.data(), m_t_w_curr.data(), pc_in.data(), pc_in.size(), LL_FMT_PCL32, LL_HOST, out.data()));
    pt_out = to_cloud(out); return (unsigned int)pc_in.size();
  }
 private:
  Context& ctx_;
};

// ---- Scene_alignment::find_tranfrom_of_two_mappings (scene_alignment.hpp:269-353) from the four feature clouds on ------------------------
class Scene_alignment {
 public:
  float m_line_res = 0.4f, m_plane_res = 0.4f, m_accepted_threshold = 0.2f;
  int m_para_scene_alignments_maximum_residual_block = 5000, m_maximum_icp_iteration = 10, m_rand_seed = 0;
  std::array<double, 4> m_q_w_curr{{1, 0, 0, 0}};   // m_pc_reg.m_q_w_curr / m_t_w_curr after the call: keyframe b into keyframe a
  std::array<double, 3> m_t_w_curr{{0, 0, 0}};
  ll_reg_result m_last{}; int m_scales_run = 0;
  explicit Scene_alignment(Context& ctx) : ctx_(ctx) {}
  // returns m_pc_reg.m_inlier_threshold (the loop-closure score; the reference truncates it to int at :390)
  double find_tranfrom_of_two_mappings(const PointCloud& source_line, const PointCloud& source_plane, const PointCloud& target_line, const PointCloud& target_plane,
                                       const std::array<double, 3>& center_a_minus_center_b) {
    ll_align_cfg c; ll_align_cfg_default(&c);
    c.line_res = m_line_res; c.plane_res = m_plane_res; c.accepted_threshold = m_accepted_threshold; c.maximum_icp_iteration = m_maximum_icp_iteration;
    c.maximum_residual_block = m_para_scene_alignments_maximum_residual_block; c.rng_seed = m_rand_seed;
    for (int k = 0; k < 3; k++) c.t_init[k] = center_a_minus_center_b[k];
    ctx_.check(ll_scene_align(ctx_.get(), source_line.data(), source_line.size(), source_plane.data(), source_plane.size(), target_line.data(), target_line.size(),
                              target_plane.data(), target_plane.size(), LL_FMT_PCL32, LL_HOST, &c, &m_last, &m_scales_run));
    for (int k = 0; k < 4; k++) m_q_w_curr[k] = m_last.q_w_curr[k];
    for (int k = 0; k < 3; k++) m_t_w_curr[k] = m_last.t_w_curr[k];
    return m_last.inlier_threshold;
  }
 private:
  Context& ctx_;
};

// ---- Points_cloud_map (cell_map_keyframe.hpp:264) as the matching path uses it -------------------------------------
class Points_cloud_map {
 public:
  explicit Points_cloud_map(Context& ctx, float resolution = 1.0f, int minimum_revisit_threshold = 2000, int max_cells = 0) : ctx_(ctx) {
    ctx_.check(ll_cellmap_create(ctx_.get(), resolution, minimum_revisit_threshold, max_cells, &map_));   // set_resolution (:674-679) + m_minimum_revisit_threshold
  }
  ~Points_cloud_map() { ll_cellmap_release(map_); }
  Points_cloud_map(const Points_cloud_map&) = delete; Points_cloud_map& operator=(const Points_cloud_map&) = delete;
  void reserve(size_t store_points, size_t scan_points = 0) { ctx_.check(ll_cellmap_reserve(ctx_.get(), map_, store_points, scan_points)); }   // no reallocation below that
  void append_cloud(const PointCloud& pts) { ctx_.check(ll_cellmap_append(ctx_.get(), map_, pts.data(), pts.size(), LL_FMT_PCL32, LL_HOST)); }   // :619-672
  int get_cells_size() const { int c = 0, p = 0, f = 0; ctx_.check(ll_cellmap_stats(ctx_.get(), map_, &c, &p, &f)); return c; }
  // update_buff_for_matching, matching_mode 1, for this map (laser_mapping.hpp:475-516): cells within search_range of t_w_curr and in the FOV,
  // each down-sampled (and replaced when down_sample_replace), concatenated in ascending cell-index order
  PointCloud cells_in_fov_downsampled(const std::array<double, 4>& q_w_curr, const std::array<double, 3>& t_w_curr, float search_range, float fov_deg, float leaf,
                                      bool down_sample_replace = true, int* cells_in_fov = nullptr) {
    int c = 0, p = 0, f = 0; ctx_.check(ll_cellmap_stats(ctx_.get(), map_, &c, &p, &f));
    std::vector<ll_point> out((size_t)(p > 0 ? p : 1)); size_t n = 0;
    ctx_.check(ll_cellmap_assemble(ctx_.get(), map_, q_w_curr.data(), t_w_curr.data(), search_range, fov_deg, leaf, down_sample_replace ? 1 : 0, out.data(), out.size(), &n, cells_in_fov, nullptr));
    out.resize(n); return to_cloud(out);
  }
  ll_cellmap* get() const { return map_; }
 private:
  Context& ctx_; ll_cellmap* map_ = nullptr;
};

// ---- Laser_mapping::process_new_scan with everything on the device (laser_mapping.hpp:1316-1521 + :460-566, matching_mode 0 and 1) ----
class Laser_mapping {
 public:
  explicit Laser_mapping(Context& ctx, const ll_mapper_config* cfg = nullptr) : ctx_(ctx) {
    if (cfg) cfg_ = *cfg; else ll_mapper_config_default(&cfg_);
    ctx_.check(ll_mapper_create(ctx_.get(), &cfg_, &mapper_));
  }
  ~Laser_mapping() { ll_mapper_release(mapper_); }
  Laser_mapping(const Laser_mapping&) = delete; Laser_mapping& operator=(const Laser_mapping&) = delete;
  // one raw scan (what Laser_feature::laserCloudHandler receives); returns the int of find_out_incremental_transfrom
  int process_new_scan(const PointCloud& raw, double time_stamp, ll_reg_result* result = nullptr, ll_mapper_stats* stats = nullptr) {
    ll_reg_result r; ll_mapper_stats st;
    ctx_.check(ll_mapper_process_scan(mapper_, raw.data(), raw.size(), LL_FMT_PCL32, LL_HOST, time_stamp, &r, &st));
    ctx_.check(ll_mapper_pose(mapper_, m_q_w_curr.data(), m_t_w_curr.data(), &m_current_frame_index));
    if (result) *result = r; if (stats) *stats = st;
    return r.status;
  }
  std::array<double, 4> m_q_w_curr{{1, 0, 0, 0}};   // (w, x, y, z)
  std::array<double, 3> m_t_w_curr{{0, 0, 0}};
  int m_current_frame_index = 0;
 private:
  Context& ctx_; ll_mapper_config cfg_; ll_mapper* mapper_ = nullptr;
};

}  // namespace ll200
