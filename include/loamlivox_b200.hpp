// loamlivox_b200.hpp — header-only C++ mirror of the reference's classes for the hot path, over the C-ABI (loamlivox_b200.h).
// Same names, argument meaning and return conventions as
//   Livox_laser                      loam_livox/source/livox_feature_extractor.hpp:77   (extract_laser_features :722, get_features :219)
//   Point_cloud_registration         loam_livox/source/point_cloud_registration.hpp:38  (find_out_incremental_transfrom :163/:585,
//                                                                                               pointcloudAssociateToMap :673)
//   Points_cloud_map                 loam_livox/source/cell_map_keyframe.hpp:264        (append_cloud :619, cells in radius + FOV :761, laser_mapping.hpp:475-516)
//   Laser_mapping::process_new_scan  loam_livox/source/laser_mapping.hpp:1316
//   Maps_keyframe                    loam_livox/source/cell_map_keyframe.hpp:1002   (analyze :1488, extract_specify_points :1263, get_center :1292,
//                                                                                               max_similiarity_of_two_image :1157)
// so that laser_feature_extractor.hpp / laser_mapping.hpp can switch with the small adapter shown in INTEGRATION.md.
// No PCL / Eigen / Ceres needed: clouds are std::vector<ll200::PointXYZI> (layout-identical to pcl::PointXYZI, 32 bytes).
#pragma once
#include <algorithm>
#include <array>
#include <cstdint>
#include <cstring>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
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
  // Several independent registrations against one map in one call (ll_register_batch): clouds[i] = (corner, surface) features of item i,
  // states[i] its parameters and initial pose.  results[i] / item_status[i] are what ll_register would return for item i alone (LL_OK, or
  // LL_ERR_NO_BLOCKS for an item that dropped out); the gpu_ms_* fields time the whole batch.  An error of the whole call throws.
  void register_batch(const Match_map& map, const std::vector<std::pair<const PointCloud*, const PointCloud*>>& clouds, const std::vector<ll_reg_state>& states,
                      std::vector<ll_reg_result>& results, std::vector<int>& item_status) {
    if (clouds.size() != states.size()) throw Error(LL_ERR_INVALID, "one state per item");
    const size_t n = clouds.size();
    std::vector<const void*> c(n), s(n); std::vector<size_t> nc(n), ns(n);
    for (size_t i = 0; i < n; i++) { c[i] = clouds[i].first->data(); nc[i] = clouds[i].first->size(); s[i] = clouds[i].second->data(); ns[i] = clouds[i].second->size(); }
    results.assign(n, ll_reg_result{}); item_status.assign(n, LL_OK);
    ctx_.check(ll_register_batch(ctx_.get(), map.get(), (int)n, c.data(), nc.data(), s.data(), ns.data(), LL_FMT_PCL32, LL_HOST, states.data(), results.data(), item_status.data()));
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

class Laser_feature;

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
  // one sensor frame (one raw cloud per head; Mid-100: 3) cut into pieces, each piece registered as a scan (odom_mode 1, the shipped configs;
  // 0: piece 0 only).  One entry per published piece in results / stats (empty when no head has more than 5 petals).
  void process_new_frame(const std::vector<PointCloud>& heads, const std::vector<double>& time_stamps, int odom_mode = 1,
                         std::vector<ll_reg_result>* results = nullptr, std::vector<ll_mapper_stats>* stats = nullptr) {
    if (heads.size() != time_stamps.size()) throw Error(LL_ERR_INVALID, "one time stamp per head");
    std::vector<const void*> raws; std::vector<size_t> ns;
    for (const PointCloud& h : heads) { raws.push_back(h.data()); ns.push_back(h.size()); }
    std::vector<ll_reg_result> r(LL_MAX_PIECES_PER_FRAME); std::vector<ll_mapper_stats> st(LL_MAX_PIECES_PER_FRAME); int n = 0;
    ctx_.check(ll_mapper_process_frame(mapper_, (int)heads.size(), raws.data(), ns.data(), LL_FMT_PCL32, LL_HOST, time_stamps.data(), odom_mode,
                                       r.data(), st.data(), (int)r.size(), &n));
    ctx_.check(ll_mapper_pose(mapper_, m_q_w_curr.data(), m_t_w_curr.data(), &m_current_frame_index));
    r.resize(n); st.resize(n);
    if (results) *results = r; if (stats) *stats = st;
  }
  // several frames of recorded data in one call: what process_new_frame returns for each in turn, the front end of frame f + 1 running on the
  // device under the registrations of frame f (heads of every frame in the same number).  results / stats: one entry per frame.  On an error
  // they hold what completed (the frames before the failing one, then its completed pieces) before Error is thrown; *done = the frames completed.
  void process_new_frames(const std::vector<std::vector<PointCloud>>& frames, const std::vector<std::vector<double>>& time_stamps, int odom_mode = 1,
                          std::vector<std::vector<ll_reg_result>>* results = nullptr, std::vector<std::vector<ll_mapper_stats>>* stats = nullptr, int* done_out = nullptr) {
    if (frames.empty() || frames.size() != time_stamps.size()) throw Error(LL_ERR_INVALID, "one list of time stamps per frame");
    const size_t nh = frames[0].size(), cap = LL_MAX_PIECES_PER_FRAME;
    std::vector<const void*> raws; std::vector<size_t> ns; std::vector<double> stamps;
    for (size_t f = 0; f < frames.size(); f++) {
      if (frames[f].size() != nh || time_stamps[f].size() != nh) throw Error(LL_ERR_INVALID, "the same heads in every frame, one time stamp per head");
      for (size_t h = 0; h < nh; h++) { raws.push_back(frames[f][h].data()); ns.push_back(frames[f][h].size()); stamps.push_back(time_stamps[f][h]); }
    }
    std::vector<ll_reg_result> r(frames.size() * cap); std::vector<ll_mapper_stats> st(frames.size() * cap); std::vector<int> n(frames.size()); int done = 0;
    const int status = ll_mapper_process_frames(mapper_, (int)frames.size(), (int)nh, raws.data(), ns.data(), LL_FMT_PCL32, LL_HOST, stamps.data(), odom_mode,
                                                r.data(), st.data(), (int)cap, n.data(), &done);
    const size_t kept = status == LL_OK ? frames.size() : std::min(frames.size(), (size_t)done + 1);
    if (results) { results->clear(); for (size_t f = 0; f < kept; f++) results->emplace_back(r.begin() + f * cap, r.begin() + f * cap + n[f]); }
    if (stats) { stats->clear(); for (size_t f = 0; f < kept; f++) stats->emplace_back(st.begin() + f * cap, st.begin() + f * cap + n[f]); }
    if (done_out) *done_out = done;
    ctx_.check(ll_mapper_pose(mapper_, m_q_w_curr.data(), m_t_w_curr.data(), &m_current_frame_index));
    ctx_.check(status);
  }
  // several raw scans of recorded data in one call: what process_new_scan returns for each in turn, the front end of scan k + 1 under the
  // mapper step of scan k.  Returns the int of find_out_incremental_transfrom per scan.  On an error results / stats hold the scans completed
  // before Error is thrown; *done = their number.
  std::vector<int> process_new_scans(const std::vector<PointCloud>& raws, const std::vector<double>& time_stamps, std::vector<ll_reg_result>* results = nullptr,
                                     std::vector<ll_mapper_stats>* stats = nullptr, int* done_out = nullptr) {
    if (raws.empty() || raws.size() != time_stamps.size()) throw Error(LL_ERR_INVALID, "one time stamp per scan");
    std::vector<const void*> ptrs; std::vector<size_t> ns;
    for (const PointCloud& c : raws) { ptrs.push_back(c.data()); ns.push_back(c.size()); }
    std::vector<ll_reg_result> r(raws.size()); std::vector<ll_mapper_stats> st(raws.size()); int done = 0;
    const int rc = ll_mapper_process_scans(mapper_, (int)raws.size(), ptrs.data(), ns.data(), LL_FMT_PCL32, LL_HOST, time_stamps.data(), r.data(), st.data(), &done);
    r.resize(rc == LL_OK ? raws.size() : (size_t)done); st.resize(r.size());
    if (results) *results = r; if (stats) *stats = st;
    if (done_out) *done_out = done;
    ctx_.check(ll_mapper_pose(mapper_, m_q_w_curr.data(), m_t_w_curr.data(), &m_current_frame_index));
    ctx_.check(rc);
    std::vector<int> status; for (const ll_reg_result& x : r) status.push_back(x.status);
    return status;
  }
  // one spinning-lidar sweep through `front`'s Velodyne front end into this mapper (ll_mapper_process_sweep: less sharp -> corners, less flat
  // -> surfaces, the full cloud's largest intensity -> max_t); front's device clouds are then this sweep's.  Returns the registration status.
  int process_new_sweep(Laser_feature& front, const PointCloud& raw, ll_reg_result* result = nullptr, ll_mapper_stats* stats = nullptr);
  // several sweeps of recorded data in one call: what process_new_sweep returns for each in turn, the front end of sweep k + 1 under the mapper
  // step of sweep k.  On an error results / stats hold the sweeps completed before Error is thrown; *done = their number.
  std::vector<int> process_new_sweeps(Laser_feature& front, const std::vector<PointCloud>& raws, std::vector<ll_reg_result>* results = nullptr,
                                      std::vector<ll_mapper_stats>* stats = nullptr, int* done_out = nullptr);
  // the whole mapper as one byte image (ll_mapper_save; format in loamlivox_b200.h): load_from_image of it, on any context, continues bit for
  // bit as this mapper does.  The mapper is not modified.
  void save_to_image(std::vector<uint8_t>& image) const {
    size_t n = 0;
    ctx_.check(ll_mapper_save(mapper_, nullptr, 0, &n));
    image.resize(n);
    ctx_.check(ll_mapper_save(mapper_, image.data(), image.size(), &n));
  }
  // a mapper on ctx in the state of `image` (ll_mapper_load).  cfg NULL: the image's config; otherwise it may differ from it only in
  // max_cells, reserve_map_points and reserve_store_points.  A refused image throws and creates nothing.
  static std::unique_ptr<Laser_mapping> load_from_image(Context& ctx, const std::vector<uint8_t>& image, const ll_mapper_config* cfg = nullptr) {
    ll_mapper* m = nullptr;
    ctx.check(ll_mapper_load(ctx.get(), image.data(), image.size(), cfg, &m));
    std::unique_ptr<Laser_mapping> out(new Laser_mapping(ctx, m));
    ctx.check(ll_mapper_pose(m, out->m_q_w_curr.data(), out->m_t_w_curr.data(), &out->m_current_frame_index));
    return out;
  }
  // tracking-loss recovery (ll_mapper_set_recovery): cfg NULL turns it off; a bad value throws and leaves the mapper unchanged.  Recovery is not
  // part of an image: a mapper from load_from_image has it off.
  void set_recovery(const ll_recovery_cfg* cfg) { ctx_.check(ll_mapper_set_recovery(mapper_, cfg)); }
  // the recovery log entries since the last read, oldest first (ll_mapper_recovery_read); *dropped = entries overwritten unread
  std::vector<ll_recovery_step> recovery_log(int* dropped = nullptr) {
    std::vector<ll_recovery_step> out, buf(LL_RECOVERY_LOG);
    int n = 0, d = 0, total = 0;
    do {
      ctx_.check(ll_mapper_recovery_read(mapper_, buf.data(), (int)buf.size(), &n, &d));
      out.insert(out.end(), buf.begin(), buf.begin() + n); total += d;
    } while (n == (int)buf.size());
    if (dropped) *dropped = total;
    return out;
  }
  // loop closure (ll_mapper_set_loop_closure, loop_closure/if_enable_loop_closure): cfg NULL turns it off; a bad value throws and leaves the
  // mapper unchanged.  Not part of a mapper image (a mapper from load_from_image has it off): loop_save / loop_load carry it.
  void set_loop_closure(const ll_loop_closure_cfg* cfg) { ctx_.check(ll_mapper_set_loop_closure(mapper_, cfg)); }
  // the loop closure as a loop image of its own (ll_mapper_loop_save; format in loamlivox_b200.h); throws when loop closure is off
  void loop_save(std::vector<uint8_t>& image) const {
    size_t n = 0;
    ctx_.check(ll_mapper_loop_save(mapper_, nullptr, 0, &n));
    image.resize(n);
    ctx_.check(ll_mapper_loop_save(mapper_, image.data(), image.size(), &n));
  }
  // restores a loop image onto this mapper (ll_mapper_loop_load; typically one from load_from_image of the mapper image saved at the same
  // step).  cfg NULL: the image's config; otherwise it may differ from it only in max_cells and reserve_*.  A refused image throws and changes nothing.
  void loop_load(const std::vector<uint8_t>& image, const ll_loop_closure_cfg* cfg = nullptr) { ctx_.check(ll_mapper_loop_load(mapper_, image.data(), image.size(), cfg)); }
  // the loop-closure events since the last read, oldest first (ll_mapper_loop_read); *dropped = events overwritten unread
  std::vector<ll_loop_event> loop_log(int* dropped = nullptr) {
    std::vector<ll_loop_event> out, buf(LL_LOOP_LOG);
    int n = 0, d = 0, total = 0;
    do {
      ctx_.check(ll_mapper_loop_read(mapper_, buf.data(), (int)buf.size(), &n, &d));
      out.insert(out.end(), buf.begin(), buf.begin() + n); total += d;
    } while (n == (int)buf.size());
    if (dropped) *dropped = total;
    return out;
  }
  // loops after the first (ll_mapper_set_loop_policy): p NULL the default (the reference's first loop, then stop); set after set_loop_closure
  // and before the first loop, else it throws and changes nothing
  void set_loop_policy(const ll_loop_policy* p) { ctx_.check(ll_mapper_set_loop_policy(mapper_, p)); }
  // loop feedback (ll_mapper_set_loop_feedback; matching mode 0): after each loop the history windows and the pose move onto the optimized
  // trajectory.  Set after set_loop_closure and before the first loop, else it throws and changes nothing
  void set_loop_feedback(bool on) { ctx_.check(ll_mapper_set_loop_feedback(mapper_, on ? 1 : 0)); }
  // the correction applied last (q_wxyz, t) and how many were applied (ll_mapper_loop_correction_read)
  int loop_correction(double q_wxyz[4], double t[3]) {
    int n = 0;
    ctx_.check(ll_mapper_loop_correction_read(mapper_, q_wxyz, t, &n));
    return n;
  }
  // every loop edge so far, in closing order (ll_mapper_loop_edges)
  std::vector<ll_pg_edge> loop_edges() {
    int n = 0;
    ctx_.check(ll_mapper_loop_edges(mapper_, nullptr, 0, &n));
    std::vector<ll_pg_edge> out(n);
    ctx_.check(ll_mapper_loop_edges(mapper_, out.data(), n, &n));
    return out;
  }
  // the keyframe poses before (pose3d_map_ori) and after the latest optimization (temp_pose_3d_map; pose3d_map_ori past the keyframes it
  // covered), the latest loop edge; returns whether a loop is closed
  bool loop_result(std::vector<ll_pose>* poses_ori, std::vector<ll_pose>* poses_opt, ll_pg_edge* edge = nullptr) {
    int n = 0, closed = 0;
    ctx_.check(ll_mapper_loop_result(mapper_, &n, &closed, nullptr, nullptr, 0, nullptr));
    poses_ori->resize(n); poses_opt->resize(n);
    ctx_.check(ll_mapper_loop_result(mapper_, &n, &closed, poses_ori->data(), poses_opt->data(), n, edge));
    return closed != 0;
  }
  std::array<double, 4> m_q_w_curr{{1, 0, 0, 0}};   // (w, x, y, z)
  std::array<double, 3> m_t_w_curr{{0, 0, 0}};
  int m_current_frame_index = 0;
 private:
  Laser_mapping(Context& ctx, ll_mapper* m) : ctx_(ctx), mapper_(m) { ll_mapper_config_default(&cfg_); }
  Context& ctx_; ll_mapper_config cfg_; ll_mapper* mapper_ = nullptr;
};

// ---- Ceres_pose_graph_3d (ceres_pose_graph_3d.hpp:198-352), Scene_alignment::add_constrain_of_loop (scene_alignment.hpp:97-127) and
// ---- Mapping_refine::refine_pointcloud (ceres_pose_graph_3d.hpp:437-500), without Eigen: quaternions as (w, x, y, z) ----------------------
struct Pose3d { std::array<double, 4> q{{1, 0, 0, 0}}; std::array<double, 3> p{{0, 0, 0}}; };
struct Constraint3d {
  int id_begin = 0, id_end = 0; Pose3d t_be; std::array<double, 36> information{};
  Constraint3d() { for (int k = 0; k < 6; k++) information[7 * k] = 1.0; }
};
typedef std::map<int, Pose3d> MapOfPoses;   // keyframe order: ids 0 .. n-1
typedef std::vector<Constraint3d> VectorOfConstraints;

class Pose_graph {
 public:
  Pose_graph(Context& ctx, int reserve_nodes = 1024, int reserve_edges = 2048) : ctx_(ctx) { ctx_.check(ll_pose_graph_create(ctx.get(), reserve_nodes, reserve_edges, &pg_)); }
  ~Pose_graph() { ll_pose_graph_release(pg_); }
  Pose_graph(const Pose_graph&) = delete; Pose_graph& operator=(const Pose_graph&) = delete;
  // pose_graph_optimization(poses, constraints): poses optimized in place; the lowest id is held constant, as SetParameterBlockConstant on poses->begin()
  ll_pg_summary pose_graph_optimization(MapOfPoses& poses, const VectorOfConstraints& constraints, int max_iterations = 200) {
    std::vector<ll_pose> x; x.reserve(poses.size());
    int expect = 0;
    for (const auto& kv : poses) {
      if (kv.first != expect++) throw Error(LL_ERR_INVALID, "pose ids must be 0 .. n-1");
      ll_pose p; for (int k = 0; k < 4; k++) p.q_wxyz[k] = kv.second.q[k]; for (int k = 0; k < 3; k++) p.t[k] = kv.second.p[k];
      x.push_back(p);
    }
    std::vector<ll_pg_edge> e(constraints.size());
    for (size_t i = 0; i < constraints.size(); i++) {
      const Constraint3d& c = constraints[i];
      e[i].id_begin = c.id_begin; e[i].id_end = c.id_end;
      for (int k = 0; k < 4; k++) e[i].q_wxyz[k] = c.t_be.q[k]; for (int k = 0; k < 3; k++) e[i].t[k] = c.t_be.p[k];
      for (int k = 0; k < 36; k++) e[i].information[k] = c.information[k];
    }
    ll_pg_summary s;
    ctx_.check(ll_pose_graph_optimize(pg_, x.data(), (int)x.size(), e.empty() ? nullptr : e.data(), (int)e.size(), max_iterations, &s));
    for (auto& kv : poses) { for (int k = 0; k < 4; k++) kv.second.q[k] = x[kv.first].q_wxyz[k]; for (int k = 0; k < 3; k++) kv.second.p[k] = x[kv.first].t[k]; }
    return s;
  }
  // Scene_alignment::add_constrain_of_loop(s_idx, t_idx, q_a, t_a, q_b, t_b, icp_q, icp_t) with laser_mapping.hpp:1065-1066's inversion of the
  // ll_scene_align pose (icp) first: the edge runs from id_b (the newer keyframe) to id_a (the older one)
  static Constraint3d add_constrain_of_loop(int id_b, int id_a, const Pose3d& a, const Pose3d& b, const std::array<double, 4>& icp_q, const std::array<double, 3>& icp_t) {
    ll_pose pa, pb; ll_pg_edge e;
    for (int k = 0; k < 4; k++) { pa.q_wxyz[k] = a.q[k]; pb.q_wxyz[k] = b.q[k]; }
    for (int k = 0; k < 3; k++) { pa.t[k] = a.p[k]; pb.t[k] = b.p[k]; }
    ll_pose_graph_loop_edge(icp_q.data(), icp_t.data(), &pa, id_a, &pb, id_b, &e);
    Constraint3d c; c.id_begin = e.id_begin; c.id_end = e.id_end;
    for (int k = 0; k < 4; k++) c.t_be.q[k] = e.q_wxyz[k]; for (int k = 0; k < 3; k++) c.t_be.p[k] = e.t[k];
    for (int k = 0; k < 36; k++) c.information[k] = e.information[k];
    return c;
  }
 private:
  Context& ctx_; ll_pose_graph* pg_ = nullptr;
};

// Mapping_refine::refine_pointcloud with if_save == 0 for every keyframe (at most 256 per call): VoxelGrid at leaf, then the float re-pose
inline std::vector<PointCloud> refine_pointclouds(Context& ctx, const std::vector<PointCloud>& clouds, const MapOfPoses& ori, const MapOfPoses& opt, float leaf) {
  std::vector<ll_point> in; std::vector<size_t> ends; std::vector<ll_pose> po, pp;
  for (const PointCloud& c : clouds) { for (const PointXYZI& p : c) in.push_back({p.x, p.y, p.z, p.intensity}); ends.push_back(in.size()); }
  for (size_t k = 0; k < clouds.size(); k++) {
    const Pose3d &a = ori.at((int)k), &b = opt.at((int)k); ll_pose x, y;
    for (int j = 0; j < 4; j++) { x.q_wxyz[j] = a.q[j]; y.q_wxyz[j] = b.q[j]; } for (int j = 0; j < 3; j++) { x.t[j] = a.p[j]; y.t[j] = b.p[j]; }
    po.push_back(x); pp.push_back(y);
  }
  std::vector<ll_point> out(in.size()); std::vector<size_t> cnt(clouds.size());
  ctx.check(ll_keyframes_repose(ctx.get(), in.data(), in.size(), ends.data(), (int)clouds.size(), po.data(), pp.data(), leaf, out.data(), cnt.data()));
  std::vector<PointCloud> res(clouds.size()); size_t w = 0;
  for (size_t k = 0; k < clouds.size(); k++) { res[k] = to_cloud(std::vector<ll_point>(out.begin() + w, out.begin() + w + cnt[k])); w += cnt[k]; }
  return res;
}

// ---- Maps_keyframe (cell_map_keyframe.hpp:1002-1494) over the cells of a full-resolution Points_cloud_map --------------------------
enum Feature_type { e_feature_sphere = LL_CELL_SPHERE, e_feature_line = LL_CELL_LINE, e_feature_plane = LL_CELL_PLANE };
class Maps_keyframe {
 public:
  explicit Maps_keyframe(Context& ctx) : ctx_(ctx) { ctx_.check(ll_keyframe_create(ctx_.get(), &kf_)); }
  ~Maps_keyframe() { ll_keyframe_release(kf_); }
  Maps_keyframe(const Maps_keyframe&) = delete; Maps_keyframe& operator=(const Maps_keyframe&) = delete;
  // m_pt_cell_map_full.append_cloud(pts, &cell_vec), then add_cells(cell_vec) on every open keyframe (laser_mapping.hpp:1527-1533)
  static void append_cloud(Context& ctx, Points_cloud_map& full, const PointCloud& pts, const std::vector<Maps_keyframe*>& open) {
    std::vector<ll_keyframe*> h; for (Maps_keyframe* k : open) h.push_back(k->kf_);
    ctx.check(ll_keyframe_append(ctx.get(), full.get(), pts.data(), pts.size(), LL_FMT_PCL32, LL_HOST, h.data(), (int)h.size()));
  }
  // analyze (:1487-1494) over the cells as `full` holds them now; if_update_mean_and_cov_incrementally is the map's setting
  int analyze(Points_cloud_map& full, int if_update_mean_and_cov_incrementally = 0) {
    ctx_.check(ll_keyframe_analyze(ctx_.get(), full.get(), kf_, if_update_mean_and_cov_incrementally, &info_)); return 0;
  }
  PointCloud extract_specify_points(Feature_type select_type) const { return cloud(select_type); }   // :1263-1280
  PointCloud get_all_pointcloud() const { return cloud(LL_CELL_ALL); }                                // :1282-1290
  std::array<float, 3> get_center() const { return {{info_.center[0], info_.center[1], info_.center[2]}}; }   // :1292-1302
  const ll_keyframe_info& info() const { return info_; }   // m_roi_range, m_ratio_nonzero_*, cell and point counts
  // max_similiarity_of_two_image(img_a, img_b) (:1157-1202) of keyframe a's and keyframe b's line or plane image, as ll_loop_search computes it
  static float max_similiarity_of_two_image(Context& ctx, const Maps_keyframe& a, const Maps_keyframe& b, Feature_type which) {
    const ll_keyframe* kfs[2] = {b.kf_, a.kf_};
    ll_loop_cfg cfg; ll_loop_cfg_default(&cfg);
    float sp = 0.f, sl = 0.f; int n = 0;
    ctx.check(ll_loop_search(ctx.get(), kfs, 2, 1, &cfg, &sp, &sl, nullptr, &n));
    return which == e_feature_line ? sl : sp;
  }
  ll_keyframe* get() const { return kf_; }
 private:
  PointCloud cloud(int which) const {
    size_t n = 0; const ll_point* dev = nullptr;
    ctx_.check(ll_keyframe_cloud(ctx_.get(), kf_, which, nullptr, 0, &n, &dev));
    std::vector<ll_point> out(n);
    if (n) ctx_.check(ll_keyframe_cloud(ctx_.get(), kf_, which, out.data(), n, &n, &dev));
    return to_cloud(out);
  }
  Context& ctx_; ll_keyframe* kf_ = nullptr; ll_keyframe_info info_ = {};
};
// service_loop_detection's candidate search (laser_mapping.hpp:988-1033) for keyframes[newest]: the candidates his ascending
inline std::vector<int> loop_search(Context& ctx, const std::vector<Maps_keyframe*>& keyframes, int newest, const ll_loop_cfg& cfg) {
  std::vector<const ll_keyframe*> h; for (Maps_keyframe* k : keyframes) h.push_back(k->get());
  std::vector<int> cand((size_t)(newest > 0 ? newest : 1)); int n = 0;
  ctx.check(ll_loop_search(ctx.get(), h.data(), (int)h.size(), newest, &cfg, nullptr, nullptr, cand.data(), &n));
  cand.resize(n); return cand;
}

// Laser_feature's Velodyne branch (laser_feature_extractor.hpp:393-825, scan_line 16 or 64) on the device: laserCloudHandler(cloud) fills
// the five clouds the reference publishes (/laser_points_2, /laser_cloud_sharp, /laser_cloud_less_sharp, /laser_cloud_flat,
// /laser_cloud_less_flat).  The 20-frame start-up delay stays the caller's.
class Laser_feature {
 public:
  Laser_feature(Context& ctx, int scan_line = 16, float minimum_range = 0.1f, float plane_resolution = 0.4f) : ctx_(ctx) {
    ll_spin_cfg cfg; ll_spin_cfg_default(&cfg);
    cfg.scan_line = scan_line; cfg.minimum_range = minimum_range; cfg.plane_resolution = plane_resolution;
    ctx_.check(ll_spin_create(ctx_.get(), &cfg, &h_));
  }
  ~Laser_feature() { ll_spin_release(h_); }
  Laser_feature(const Laser_feature&) = delete; Laser_feature& operator=(const Laser_feature&) = delete;
  void laserCloudHandler(const PointCloud& in) {
    ctx_.check(ll_spin_extract(h_, in.data(), in.size(), LL_FMT_PCL32, LL_HOST, nullptr));
    laserCloud = cloud(LL_SPIN_FULL); cornerPointsSharp = cloud(LL_SPIN_SHARP); cornerPointsLessSharp = cloud(LL_SPIN_LESS_SHARP);
    surfPointsFlat = cloud(LL_SPIN_FLAT); surfPointsLessFlat = cloud(LL_SPIN_LESS_FLAT);
  }
  // device form of cloud `which` (LL_SPIN_*), valid until the next laserCloudHandler: an LL_DEVICE input of ll_register / ll_map_build
  const ll_point* device_cloud(int which, size_t* n) const { const ll_point* d = nullptr; ctx_.check(ll_spin_cloud(h_, which, nullptr, 0, n, &d)); return d; }
  PointCloud laserCloud, cornerPointsSharp, cornerPointsLessSharp, surfPointsFlat, surfPointsLessFlat;
  ll_spin* get() const { return h_; }
 private:
  PointCloud cloud(int which) const {
    size_t n = 0;
    ctx_.check(ll_spin_cloud(h_, which, nullptr, 0, &n, nullptr));
    std::vector<ll_point> tmp(n);
    if (n) ctx_.check(ll_spin_cloud(h_, which, tmp.data(), n, &n, nullptr));
    PointCloud out(n);
    for (size_t i = 0; i < n; i++) { out[i] = PointXYZI{}; out[i].x = tmp[i].x; out[i].y = tmp[i].y; out[i].z = tmp[i].z; out[i].intensity = tmp[i].intensity; }
    return out;
  }
  Context& ctx_;
  ll_spin* h_ = nullptr;
};

inline int Laser_mapping::process_new_sweep(Laser_feature& front, const PointCloud& raw, ll_reg_result* result, ll_mapper_stats* stats) {
  ll_reg_result r; ll_mapper_stats st;
  ctx_.check(ll_mapper_process_sweep(mapper_, front.get(), raw.data(), raw.size(), LL_FMT_PCL32, LL_HOST, &r, &st));
  ctx_.check(ll_mapper_pose(mapper_, m_q_w_curr.data(), m_t_w_curr.data(), &m_current_frame_index));
  if (result) *result = r; if (stats) *stats = st;
  return r.status;
}
inline std::vector<int> Laser_mapping::process_new_sweeps(Laser_feature& front, const std::vector<PointCloud>& raws, std::vector<ll_reg_result>* results,
                                                          std::vector<ll_mapper_stats>* stats, int* done_out) {
  if (raws.empty()) throw Error(LL_ERR_INVALID, "no sweeps");
  std::vector<const void*> ptrs; std::vector<size_t> ns;
  for (const PointCloud& c : raws) { ptrs.push_back(c.data()); ns.push_back(c.size()); }
  std::vector<ll_reg_result> r(raws.size()); std::vector<ll_mapper_stats> st(raws.size()); int done = 0;
  const int rc = ll_mapper_process_sweeps(mapper_, front.get(), (int)raws.size(), ptrs.data(), ns.data(), LL_FMT_PCL32, LL_HOST, r.data(), st.data(), &done);
  r.resize(rc == LL_OK ? raws.size() : (size_t)done); st.resize(r.size());
  if (results) *results = r; if (stats) *stats = st;
  if (done_out) *done_out = done;
  ctx_.check(ll_mapper_pose(mapper_, m_q_w_curr.data(), m_t_w_curr.data(), &m_current_frame_index));
  ctx_.check(rc);
  std::vector<int> status; for (const ll_reg_result& x : r) status.push_back(x.status);
  return status;
}

}  // namespace ll200
