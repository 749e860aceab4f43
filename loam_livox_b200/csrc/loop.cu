// Loop closure inside the streaming mapper (ll_mapper_set_loop_closure; DESIGN.md §4.6): Laser_mapping::process_new_scan's keyframe block
// (loam_livox/source/laser_mapping.hpp:1442, 1446-1459, 1480-1487, 1523-1564) and service_loop_detection (:874-1127), run by the mapper step
// that appends its features, with every full cloud on the device.  Everything below is host orchestration of the library's own entry points
// (transform, VoxelGrid, ll_keyframe_*, ll_loop_search, ll_scene_align, the pose graph, the re-pose) plus one gather kernel and, with loop
// feedback on, one kernel that moves the mapper's history windows onto the optimized trajectory.
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstring>
#include "common.cuh"
#include "kernels.cuh"
#include "cellmap.cuh"
#include "exact_math.cuh"

// grid (chunks, publish x heads): the full slice of head h for piece i goes to segment i after the slices of heads 0 .. h-1
// (laser_feature_extractor.hpp:353-358 sums the heads' full clouds of a piece in head order).  Block (0, 0) also writes the segment ends.
__global__ void lc_gather_full_kernel(const FrameSlices* __restrict__ sl, FrameBases B, int n_heads, int publish, const float4* __restrict__ src,
                                      float4* __restrict__ dst, int* __restrict__ seg_end) {
  const int pair = blockIdx.y, i = pair / n_heads, h = pair % n_heads;
  int o = 0;
  for (int p = 0; p < pair; p++) o += sl[p % n_heads].len[2][p / n_heads];
  const int len = sl[h].len[2][i];
  const float4* s = src + B.base[h] + sl[h].off[2][i];
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < len; k += gridDim.x * blockDim.x) dst[o + k] = s[k];
  if (blockIdx.x != 0 || pair != 0) return;
  const int t = threadIdx.x;
  if (t < publish) { int e = 0; for (int p = 0; p <= t; p++) for (int hh = 0; hh < n_heads; hh++) e += sl[hh].len[2][p]; seg_end[t] = e; }
}

// Loop feedback (DESIGN.md §4.6.2): both history windows moved in place, window w's point i (c: nc points, then s: ns points) by the delta of
// its segment, the first whose end (ends[w * n_seg ...], staged in shared memory) is past i.  delta: n_seg poses (q w, x, y, z, t), fp64 from the
// float point and rounded once, intensity kept: transform_kernel's arithmetic (qrot_d, then + t).
__global__ void lc_window_correct_kernel(float4* __restrict__ c, int nc, float4* __restrict__ s, int ns, const int* __restrict__ ends, int n_seg,
                                         const double* __restrict__ delta) {
  extern __shared__ int sh_end[];
  for (int k = threadIdx.x; k < 2 * n_seg; k += blockDim.x) sh_end[k] = ends[k];
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nc + ns) return;
  const bool surf = i >= nc;
  const int j = surf ? i - nc : i;
  const int* e = sh_end + (surf ? n_seg : 0);
  int lo = 0, hi = n_seg - 1;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (e[mid] > j) hi = mid; else lo = mid + 1; }
  float4* p = surf ? s + j : c + j;
  const float4 v = *p;
  const double* d = delta + 7 * lo;
  const double q[4] = {d[0], d[1], d[2], d[3]};
  double wx, wy, wz; qrot_d(q, (double)v.x, (double)v.y, (double)v.z, wx, wy, wz);
  *p = make_float4((float)(wx + d[4]), (float)(wy + d[5]), (float)(wz + d[6]), v.w);
}

// feedback: the step's odometry-frame pose, then per window segment its delta (7 doubles) and both windows' segment ends
struct FeedbackLayout {
  double* pose; double* delta; int* ends;
  void layout(Carve& k, size_t n_seg) { pose = k.take<double>(7); delta = k.take<double>(7 * n_seg); ends = k.take<int>(2 * n_seg); }
};

// in: the step's full cloud (a scan: the compaction's three outputs, only `full` kept; a frame: the published pieces one after another), the
// compaction's counts, the pieces' ends
struct LoopInLayout {
  float4* full; float4* junk[2]; int* cnt; int* seg_end;
  void layout(Carve& k, size_t full_pts, size_t scan_pts) {
    full = k.take<float4>(full_pts); junk[0] = k.take<float4>(scan_pts); junk[1] = k.take<float4>(scan_pts); cnt = k.take<int>(12); seg_end = k.take<int>(LL_MAX_PIECES);
  }
};
// refine: the down-sampled and the re-posed keyframe clouds, the segment ends and affines of one chunk of 256 keyframes
struct RefineLayout {
  float4* mid; float4* out; int* end; int* oend; float* aff;
  void layout(Carve& k, size_t n) { mid = k.take<float4>(n); out = k.take<float4>(n); end = k.take<int>(256); oend = k.take<int>(256); aff = k.take<float>(12 * 256); }
};

struct LoopClosure {
  ll_loop_closure_cfg cfg;
  float cell_res = 1.f; int revisit = 1, max_history = 0;
  ll_cellmap* full = nullptr;                        // m_pt_cell_map_full
  DevBuf in, world;                                  // LoopInLayout; the step's cloud in the world frame
  size_t in_full = 0, in_scan = 0;                   // LoopInLayout sizes
  std::vector<int> seg;                              // ends of the captured pieces (a scan: one)
  HistoryWindow his;                                 // m_laser_cloud_full_history
  struct Open { ll_keyframe* kf; int frames; };
  std::vector<Open> open;                            // m_keyframe_of_updating_list
  std::vector<ll_keyframe*> kfs;                     // keyframe_vec
  std::vector<ll_pose> poses;                        // pose3d_vec (= pose3d_map_ori)
  std::vector<ll_pg_edge> edges;                     // constrain_vec
  DevBuf acc; std::vector<size_t> acc_end;           // accumulated clouds, down-sampled, in keyframe order (map_id_pc)
  ll_pose_graph* pg = nullptr;
  ll_loop_policy policy{1, 0};                       // ll_mapper_set_loop_policy; the default is the reference's if_end
  bool stopped = false;                              // an error of the loop work stopped it (LL_LOOP_ERROR)
  bool seg_read = false;                             // seg holds the captured cloud's ends (read by the first step after a capture)
  int piece = 0;                                     // the step's piece of the captured frame
  std::vector<ll_pg_edge> loops;                     // every loop edge, in closing order (constrain_vec_temp.back() of each loop)
  std::vector<ll_pose> opt;                          // temp_pose_3d_map of the latest loop: its n_opt keyframes
  bool done() const { return (int)loops.size() >= policy.max_loops; }   // all loop-closure work stops (if_end after the first loop by default)
  DevBuf refine; std::vector<int> ref_end;           // RefineLayout: the re-posed clouds of every keyframe
  EventLog<ll_loop_event> log;
  // loop feedback (ll_mapper_set_loop_feedback): each closed keyframe's frame index (-1: restored from an image that does not record it), the
  // correction applied last (C) and how many were applied; fb: FeedbackLayout for maximum_history_size segments
  bool feedback = false;
  std::vector<int> kf_frame;
  ll_pose corr{{1, 0, 0, 0}, {0, 0, 0}};
  int n_applied = 0;
  DevBuf fb;
};

namespace {

const char* loop_cfg_error(const ll_loop_closure_cfg& c) {
  auto pos = [](double x) { return std::isfinite(x) && x > 0.0; };
  if (c.scans_of_each_keyframe < 1 || c.scans_between_two_keyframe < 1) return "scans_of_each_keyframe and scans_between_two_keyframe must be >= 1";
  if (c.scans_between_two_keyframe >= c.scans_of_each_keyframe) return "scans_between_two_keyframe must be < scans_of_each_keyframe";
  const ll_loop_cfg& l = c.loop;
  if (l.minimum_keyframe_differen < 0) return "minimum_keyframe_differen must be >= 0";
  const double f[] = {l.avail_ratio_plane, l.avail_ratio_line, l.maximum_roi_difference, l.minimum_similarity_linear, l.minimum_similarity_planar, l.plane_with_line};
  for (double x : f) if (!std::isfinite(x)) return "the search's gates must be finite";
  if (!pos(c.map_alignment_resolution)) return "map_alignment_resolution must be finite and > 0";
  if (c.map_alignment_maximum_icp_iteration < 1) return "map_alignment_maximum_icp_iteration must be >= 1";
  if (!pos(c.map_alignment_inlier_threshold)) return "map_alignment_inlier_threshold must be finite and > 0";
  if (c.scene_alignment_maximum_residual_block < 1) return "scene_alignment_maximum_residual_block must be >= 1";
  if (!pos(c.surround_pointcloud_resolution) || !pos((float)c.surround_pointcloud_resolution)) return "surround_pointcloud_resolution must be finite and > 0";
  if (c.incremental_cov != 0 && c.incremental_cov != 1) return "incremental_cov must be 0 or 1";
  if (c.max_cells < 0 || c.max_cells > MAX_CELLS) return "max_cells must be 0 ... 2^29";
  if (c.reserve_map_points < 0 || c.reserve_map_points > INT32_MAX || c.reserve_history_points < 0 || c.reserve_history_points > INT32_MAX)
    return "reservations must be 0 ... 2^31 - 1 points";
  if (c.reserve_keyframes < 0 || c.reserve_keyframes > (1 << 20)) return "reserve_keyframes must be 0 ... 2^20";
  return nullptr;
}

// The config field by field into zeroed storage: its padding bytes are zero whatever the caller's struct held, so the loop image (which
// holds the config verbatim) and the comparison of a load's cfg depend on the values only.
ll_loop_closure_cfg loop_cfg_canonical(const ll_loop_closure_cfg& c) {
  ll_loop_closure_cfg o; memset(&o, 0, sizeof(o));
  o.scans_of_each_keyframe = c.scans_of_each_keyframe; o.scans_between_two_keyframe = c.scans_between_two_keyframe;
  o.loop.minimum_keyframe_differen = c.loop.minimum_keyframe_differen; o.loop.avail_ratio_plane = c.loop.avail_ratio_plane;
  o.loop.avail_ratio_line = c.loop.avail_ratio_line; o.loop.maximum_roi_difference = c.loop.maximum_roi_difference;
  o.loop.minimum_similarity_linear = c.loop.minimum_similarity_linear; o.loop.minimum_similarity_planar = c.loop.minimum_similarity_planar;
  o.loop.plane_with_line = c.loop.plane_with_line;
  o.map_alignment_resolution = c.map_alignment_resolution; o.map_alignment_maximum_icp_iteration = c.map_alignment_maximum_icp_iteration;
  o.map_alignment_inlier_threshold = c.map_alignment_inlier_threshold; o.scene_alignment_maximum_residual_block = c.scene_alignment_maximum_residual_block;
  o.surround_pointcloud_resolution = c.surround_pointcloud_resolution; o.incremental_cov = c.incremental_cov; o.rng_seed = c.rng_seed;
  o.max_cells = c.max_cells; o.reserve_map_points = c.reserve_map_points; o.reserve_history_points = c.reserve_history_points;
  o.reserve_keyframes = c.reserve_keyframes;
  return o;
}

// A growing device array whose contents survive the growth (DevBuf::reserve does not keep them).
int grow_keep(ll_ctx* ctx, DevBuf& b, size_t used, size_t need) {
  if (need <= b.cap) return LL_OK;
  DevBuf nb; nb.floor = b.floor;
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  LL_CUDA(ctx, nb.reserve(std::max(need, 2 * b.cap)));
  if (used) LL_CUDA(ctx, cudaMemcpyAsync(nb.p, b.p, used, cudaMemcpyDeviceToDevice, ctx->stream));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  b.release(); b = nb; nb.p = nullptr;
  return LL_OK;
}

// ---- poses in fp64 (ll_pose: q w, x, y, z and t), as the feedback and ll_loop_correction compose them
const ll_pose IDENTITY{{1, 0, 0, 0}, {0, 0, 0}};
void qrot_h(const double* q, const double* v, double* o) {   // qrot_d's association on the host
  const double ux = q[1], uy = q[2], uz = q[3], w = q[0];
  double cx = uy * v[2] - uz * v[1], cy = uz * v[0] - ux * v[2], cz = ux * v[1] - uy * v[0];
  cx = cx + cx; cy = cy + cy; cz = cz + cz;
  const double dx = uy * cz - uz * cy, dy = uz * cx - ux * cz, dz = ux * cy - uy * cx;
  o[0] = (v[0] + cx * w) + dx; o[1] = (v[1] + cy * w) + dy; o[2] = (v[2] + cz * w) + dz;
}
ll_pose compose(const ll_pose& a, const ll_pose& b) {   // a o b: (q_a q_b, R_a t_b + t_a)
  ll_pose o; quat_mul(a.q_wxyz, b.q_wxyz, o.q_wxyz);
  double r[3]; qrot_h(a.q_wxyz, b.t, r);
  for (int k = 0; k < 3; k++) o.t[k] = r[k] + a.t[k];
  return o;
}
ll_pose inverse(const ll_pose& a) {   // (q*, -(R* t))
  ll_pose o; o.q_wxyz[0] = a.q_wxyz[0]; for (int k = 1; k < 4; k++) o.q_wxyz[k] = -a.q_wxyz[k];
  double r[3]; qrot_h(o.q_wxyz, a.t, r);
  for (int k = 0; k < 3; k++) o.t[k] = -r[k];
  return o;
}
bool finite_pose(const ll_pose& p) { return finite_d(p.q_wxyz, 4) && finite_d(p.t, 3); }

// A_k = opt_k o ori_k^-1; A_0 the identity (the graph holds pose 0 constant)
ll_pose keyframe_correction(const ll_pose* ori, const ll_pose* opt, int k) { return k == 0 ? IDENTITY : compose(opt[k], inverse(ori[k])); }

// ll_loop_correction on checked inputs (f strictly ascending, n >= 1)
ll_pose correction_at(const ll_pose* ori, const ll_pose* opt, const int* f, int n, int s) {
  if (s <= f[0]) return IDENTITY;
  if (s >= f[n - 1]) return keyframe_correction(ori, opt, n - 1);
  const int k = (int)(std::upper_bound(f, f + n, s) - f) - 1;   // f[k] <= s < f[k + 1]
  const ll_pose a = keyframe_correction(ori, opt, k);
  if (s == f[k]) return a;
  const ll_pose b = keyframe_correction(ori, opt, k + 1);
  const double u = (double)(s - f[k]) / (double)(f[k + 1] - f[k]);
  // slerp along the shorter arc: theta the angle between the quaternions as 4-vectors, 2 atan2(|a - b|, |a + b|)
  double qb[4], dot = 0, dn = 0, sn = 0;
  for (int j = 0; j < 4; j++) dot = dot + a.q_wxyz[j] * b.q_wxyz[j];
  for (int j = 0; j < 4; j++) qb[j] = dot < 0 ? -b.q_wxyz[j] : b.q_wxyz[j];
  for (int j = 0; j < 4; j++) { const double x = a.q_wxyz[j] - qb[j], y = a.q_wxyz[j] + qb[j]; dn = dn + x * x; sn = sn + y * y; }
  const double theta = 2.0 * std::atan2(std::sqrt(dn), std::sqrt(sn));
  ll_pose o;
  if (theta == 0.0) { for (int j = 0; j < 4; j++) o.q_wxyz[j] = a.q_wxyz[j]; }
  else {
    const double st = std::sin(theta), wa = std::sin((1.0 - u) * theta) / st, wb = std::sin(u * theta) / st;
    for (int j = 0; j < 4; j++) o.q_wxyz[j] = wa * a.q_wxyz[j] + wb * qb[j];
  }
  for (int j = 0; j < 3; j++) o.t[j] = a.t[j] + u * (b.t[j] - a.t[j]);
  return o;
}

ll_loop_event* log_push(LoopClosure* lc, int kind) {
  ll_loop_event* e = lc->log.push();
  e->kind = kind; e->keyframe = (int)lc->kfs.size() - 1;
  return e;
}

void free_keyframes(LoopClosure* lc) {
  for (auto& o : lc->open) ll_keyframe_release(o.kf);
  for (ll_keyframe* k : lc->kfs) ll_keyframe_release(k);
  lc->open.clear(); lc->kfs.clear();
}

// Mapping_refine::refine_pointcloud (if_save 0) of every keyframe from the accumulated clouds and both pose sets, 256 per launch chain; the
// readers give the published ones.  The loop's last step, and what ll_mapper_loop_load recomputes (the same code: the same bits).
int loop_refine(ll_ctx* ctx, LoopClosure* lc) {
  const int n = (int)lc->opt.size();   // n_opt: the keyframes of the latest optimization (later ones keep its refined clouds)
  const size_t total = lc->acc_end.empty() ? 0 : lc->acc_end[n - 1];
  RefineLayout rl; LL_CUDA(ctx, lc->refine.carve([&](Carve& k) { rl.layout(k, total); }));
  lc->ref_end.assign(n, 0);
  for (int k0 = 0; k0 < n; k0 += 256) {
    const int nk = std::min(256, n - k0);
    const size_t b0 = k0 ? lc->acc_end[k0 - 1] : 0;
    std::vector<int> ends(nk), oend(nk);
    for (int k = 0; k < nk; k++) ends[k] = (int)(lc->acc_end[k0 + k] - b0);
    LL_TRY(keyframes_repose_dev(ctx, (const float4*)lc->acc.p + b0, ends[nk - 1], ends.data(), nk, &lc->poses[k0], &lc->opt[k0], 0.2f, rl.mid + b0, rl.out + b0,
                                rl.end, rl.oend, rl.aff, oend.data()));
    for (int k = 0; k < nk; k++) lc->ref_end[k0 + k] = (int)b0 + oend[k];   // keyframe k's output: [b0 + oend[k - 1], b0 + oend[k])
  }
  return LL_OK;
}

// Loop feedback after a loop (DESIGN.md §4.6.2): prev holds the previous loop's optimized poses, lc->opt this loop's.  Everything is computed
// and checked on the host before the one upload and the one launch; the mapper's host state moves after them.
int feedback_apply(ll_ctx* ctx, LoopClosure* lc, const std::vector<ll_pose>& prev, const MapperWindow& mw) {
  const int n = (int)lc->opt.size(), np = lc->n_applied ? (int)prev.size() : 0;
  const std::vector<int>& fr = *mw.frame;
  const int S = (int)fr.size();
  const HistoryWindow& hc = *mw.his[0]; const HistoryWindow& hs = *mw.his[1];
  if ((size_t)S != hc.segs.size() || (size_t)S != hs.segs.size()) { ctx->set_error("loop feedback: window segments and their frame indices disagree"); return LL_ERR_INVALID; }
  if (S > lc->max_history) { ctx->set_error("loop feedback: more window segments than maximum_history_size"); return LL_ERR_INVALID; }
  if (hc.live() + hs.live() > (size_t)INT32_MAX) { ctx->set_error("loop feedback: more than 2^31 - 1 window points"); return LL_ERR_INVALID; }
  for (int k = 0; k < n; k++) if (lc->kf_frame[k] < 0 || (k && lc->kf_frame[k] <= lc->kf_frame[k - 1])) { ctx->set_error("loop feedback: keyframe frame indices"); return LL_ERR_INVALID; }
  std::vector<double> delta(7 * (size_t)S);
  std::vector<int> ends(2 * (size_t)S);
  for (int i = 0; i < S; i++) {
    const ll_pose a = correction_at(lc->poses.data(), lc->opt.data(), lc->kf_frame.data(), n, fr[i]);
    const ll_pose b = np ? correction_at(lc->poses.data(), prev.data(), lc->kf_frame.data(), np, fr[i]) : IDENTITY;
    const ll_pose d = compose(a, inverse(b));
    if (!finite_pose(d)) { ctx->set_error("loop feedback: non-finite correction"); return LL_ERR_INVALID; }
    memcpy(&delta[7 * (size_t)i], d.q_wxyz, 4 * sizeof(double)); memcpy(&delta[7 * (size_t)i + 4], d.t, 3 * sizeof(double));
    ends[i] = (int)(hc.segs[i].first + hc.segs[i].second - hc.head()); ends[S + i] = (int)(hs.segs[i].first + hs.segs[i].second - hs.head());
  }
  const ll_pose a_new = keyframe_correction(lc->poses.data(), lc->opt.data(), n - 1);
  ll_pose last; memcpy(last.q_wxyz, mw.last_q, sizeof(last.q_wxyz)); memcpy(last.t, mw.last_t, sizeof(last.t));
  last = compose(compose(a_new, inverse(lc->corr)), last);   // the last addition was in the frame of the previous correction
  if (!finite_pose(a_new) || !finite_pose(last) || !finite_pose(lc->opt[n - 1])) { ctx->set_error("loop feedback: non-finite correction"); return LL_ERR_INVALID; }
  const int nc = (int)hc.live(), ns = (int)hs.live();
  if (S > 0 && nc + ns > 0) {
    cudaStream_t s = ctx->stream;
    FeedbackLayout fl; LL_CUDA(ctx, lc->fb.carve([&](Carve& k) { fl.layout(k, (size_t)S); }));   // (reserved: no reallocation)
    LL_CUDA(ctx, cudaMemcpyAsync(fl.delta, delta.data(), delta.size() * sizeof(double), cudaMemcpyHostToDevice, s));
    LL_CUDA(ctx, cudaMemcpyAsync(fl.ends, ends.data(), ends.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    lc_window_correct_kernel<<<ll_div_up(nc + ns, 256), 256, 2 * S * sizeof(int), s>>>((float4*)hc.data(), nc, (float4*)hs.data(), ns, fl.ends, S, fl.delta);
    ctx->launches++;
    LL_CUDA(ctx, cudaGetLastError());
  }
  memcpy(mw.q, lc->opt[n - 1].q_wxyz, 4 * sizeof(double)); memcpy(mw.t, lc->opt[n - 1].t, 3 * sizeof(double));
  memcpy(mw.last_q, last.q_wxyz, 4 * sizeof(double)); memcpy(mw.last_t, last.t, 3 * sizeof(double));
  *mw.map_dirty = true;
  lc->corr = a_new; lc->n_applied++;
  return LL_OK;
}

// The feedback's device buffer for maximum_history_size segments, so that no step allocates it.
int feedback_reserve(ll_ctx* ctx, LoopClosure* lc) {
  cudaSetDevice(ctx->device);
  FeedbackLayout fl; LL_CUDA(ctx, lc->fb.reserve_floor(layout_bytes([&](Carve& k) { fl.layout(k, (size_t)std::max(lc->max_history, 0)); })));
  return LL_OK;
}

// The candidates of the newest keyframe (ll_loop_search's, his ascending) through the alignment with the skips of :1048-1052 and
// :1113-1116, and on a loop the graph, the refined clouds (:1056-1100) and, with loop feedback on, the correction of the mapper.
int loop_align(ll_ctx* ctx, LoopClosure* lc, const std::vector<int>& cand, const MapperWindow& mw) {
  const ll_loop_closure_cfg& c = lc->cfg;
  const int n = (int)lc->kfs.size(), newest = n - 1;
  ll_align_cfg acfg; ll_align_cfg_default(&acfg);
  acfg.line_res = acfg.plane_res = c.map_alignment_resolution; acfg.maximum_icp_iteration = c.map_alignment_maximum_icp_iteration;
  acfg.maximum_residual_block = c.scene_alignment_maximum_residual_block; acfg.accepted_threshold = c.map_alignment_inlier_threshold; acfg.rng_seed = c.rng_seed;
  const double thr = (double)c.map_alignment_inlier_threshold, thr2 = (double)(c.map_alignment_inlier_threshold * 2);   // float parameter, double score
  int skip_to = -1;
  for (const int his : cand) {
    if (his <= skip_to) continue;
    const ll_point *sl, *sp, *tl, *tp; size_t nsl, nsp, ntl, ntp;
    LL_TRY(ll_keyframe_cloud(ctx, lc->kfs[newest], LL_CELL_LINE, nullptr, 0, &nsl, &sl));
    LL_TRY(ll_keyframe_cloud(ctx, lc->kfs[newest], LL_CELL_PLANE, nullptr, 0, &nsp, &sp));
    LL_TRY(ll_keyframe_cloud(ctx, lc->kfs[his], LL_CELL_LINE, nullptr, 0, &ntl, &tl));
    LL_TRY(ll_keyframe_cloud(ctx, lc->kfs[his], LL_CELL_PLANE, nullptr, 0, &ntp, &tp));
    ll_keyframe_info a, b; LL_TRY(ll_keyframe_get_info(lc->kfs[newest], &a)); LL_TRY(ll_keyframe_get_info(lc->kfs[his], &b));
    for (int k = 0; k < 3; k++) acfg.t_init[k] = (double)(a.center[k] - b.center[k]);   // float difference, then double (scene_alignment.hpp:303)
    ll_reg_result r; int scales = 0;
    const int sa = ll_scene_align(ctx, sl, nsl, sp, nsp, tl, ntl, tp, ntp, LL_FMT_XYZI16, LL_DEVICE, &acfg, &r, &scales);
    if (sa == LL_ERR_CUDA) return sa;
    ll_loop_event* e = log_push(lc, LL_LOOP_ALIGNMENT);
    e->his = his;
    if (sa != LL_OK) { e->decision = LL_LOOP_FAILED; e->status = sa; return LL_OK; }
    e->scales_run = scales; e->inlier_threshold = r.inlier_threshold;
    for (int k = 0; k < 4; k++) e->icp_q_wxyz[k] = r.q_w_curr[k];
    for (int k = 0; k < 3; k++) e->icp_t[k] = r.t_w_curr[k];
    if (r.inlier_threshold > thr2) { e->decision = LL_LOOP_SKIP10; skip_to = his + 10; continue; }
    if (!(r.inlier_threshold < thr)) { e->decision = LL_LOOP_SKIP5; skip_to = his + 5; continue; }
    e->decision = LL_LOOP_ACCEPT;
    // the loop (:1056-1100): the edge, the graph on the odometry edges plus every loop edge so far (the reference's one loop: this one only),
    // solved from poses_ori, the refined clouds
    ll_pg_edge le;
    ll_pose_graph_loop_edge(r.q_w_curr, r.t_w_curr, &lc->poses[his], his, &lc->poses[newest], newest, &le);
    std::vector<ll_pg_edge> edges = lc->edges; edges.insert(edges.end(), lc->loops.begin(), lc->loops.end()); edges.push_back(le);
    std::vector<ll_pose> opt = lc->poses;
    ll_pg_summary sum;
    LL_TRY(ll_pose_graph_optimize(lc->pg, opt.data(), n, edges.data(), (int)edges.size(), 200, &sum));
    lc->opt.swap(opt);
    LL_TRY(loop_refine(ctx, lc));
    lc->loops.push_back(le);
    ll_loop_event* ce = log_push(lc, LL_LOOP_CLOSED);
    ce->his = his; ce->edge = le; ce->summary = sum;
    if (lc->feedback) LL_TRY(feedback_apply(ctx, lc, opt, mw));   // (opt: the previous loop's poses after the swap)
    return LL_OK;
  }
  return LL_OK;
}

}  // namespace

int loop_set(ll_ctx* ctx, LoopClosure** plc, const ll_loop_closure_cfg* cfg, const ll_mapper_config& mcfg, int pieces) {
  if (!cfg) { loop_release(*plc); *plc = nullptr; return LL_OK; }
  if (const char* err = loop_cfg_error(*cfg)) { ctx->set_error(std::string("loop closure config: ") + err); return LL_ERR_INVALID; }
  cudaSetDevice(ctx->device);
  LoopClosure* lc = new LoopClosure();
  lc->cfg = loop_cfg_canonical(*cfg); lc->cell_res = mcfg.cell_resolution; lc->revisit = mcfg.threshold_cell_revisit; lc->max_history = mcfg.maximum_history_size;
  const int st = [&]() -> int {
    const size_t S = (size_t)ctx->cfg.max_scan_points;
    LL_TRY(ll_cellmap_create(ctx, lc->cell_res, lc->revisit, cfg->max_cells, &lc->full));
    if (cfg->reserve_map_points > 0) LL_TRY(ll_cellmap_reserve(ctx, lc->full, (size_t)cfg->reserve_map_points, S));
    lc->in_full = (size_t)std::max(pieces, 1) * S; lc->in_scan = S;
    LoopInLayout il; LL_CUDA(ctx, lc->in.reserve_floor(layout_bytes([&](Carve& k) { il.layout(k, lc->in_full, lc->in_scan); })));
    LL_CUDA(ctx, lc->world.reserve_floor(S * 16));
    if (cfg->reserve_history_points > 0) {
      LL_TRY(lc->his.reserve(ctx, (size_t)cfg->reserve_history_points));
      LL_CUDA(ctx, lc->acc.reserve_floor((size_t)cfg->reserve_history_points * 16));
    }
    const int K = std::max(cfg->reserve_keyframes, 2);
    LL_TRY(ll_pose_graph_create(ctx, K, K, &lc->pg));
    lc->kfs.reserve(K); lc->poses.reserve(K); lc->edges.reserve(K); lc->acc_end.reserve(K);
    ll_keyframe* kf = nullptr;
    LL_TRY(ll_keyframe_create(ctx, &kf));
    lc->open.push_back({kf, 0});   // :626
    lc->log.open(LL_LOOP_LOG);
    return LL_OK;
  }();
  if (st != LL_OK) { loop_release(lc); return st; }
  loop_release(*plc);
  *plc = lc;
  return LL_OK;
}

void loop_release(LoopClosure* lc) {
  if (!lc) return;
  free_keyframes(lc);
  ll_cellmap_release(lc->full);
  ll_pose_graph_release(lc->pg);
  lc->in.release(); lc->world.release(); lc->his.release(); lc->acc.release(); lc->refine.release();
  delete lc;
}

int loop_scan_cloud(ll_ctx* ctx, LoopClosure* lc, const ll_pipeline_cfg* pc) {
  if (lc->done() || lc->stopped) return LL_OK;
  cudaStream_t s = ctx->stream;
  LoopInLayout il; LL_CUDA(ctx, lc->in.carve([&](Carve& k) { il.layout(k, lc->in_full, lc->in_scan); }));
  // the front end's compaction again, on the extractor's state of this scan, keeping the full cloud (the front end keeps only the features)
  const float* d_bounds = pc->whole_frame ? nullptr : ctx->A.bounds + 2 * pc->use_piece;
  LL_TRY(launch_get_features(ctx, s, ctx->scratch, d_bounds, 0.f, 1.f, il.junk[0], il.junk[1], il.full, il.cnt));
  LL_CUDA(ctx, cudaMemcpyAsync(il.seg_end, il.cnt + 2, sizeof(int), cudaMemcpyDeviceToDevice, s));   // one segment: the full cloud
  lc->seg.assign(1, 0); lc->seg_read = false; lc->piece = 0;
  return LL_OK;
}

int loop_frame_clouds(ll_ctx* ctx, LoopClosure* lc, const FrameDev* dev, const size_t* ns, int n_heads, int publish) {
  if (lc->done() || lc->stopped) return LL_OK;
  cudaStream_t s = ctx->stream;
  LoopInLayout il; LL_CUDA(ctx, lc->in.carve([&](Carve& k) { il.layout(k, lc->in_full, lc->in_scan); }));
  FrameBases B; int base = 0, max_n = 0;
  for (int h = 0; h < n_heads; h++) { B.base[h] = base; base += (int)ns[h]; max_n = std::max(max_n, (int)ns[h]); }
  const dim3 grid(std::max(1, std::min(ll_div_up(max_n, 256 * 8), 64)), publish * n_heads);
  lc_gather_full_kernel<<<grid, 256, 0, s>>>(dev->head, B, n_heads, publish, ctx->A.tmp_c, il.full, il.seg_end); ctx->launches++;
  LL_CUDA(ctx, cudaGetLastError());
  lc->seg.assign(publish, 0); lc->seg_read = false; lc->piece = 0;
  return LL_OK;
}

int loop_sweep_cloud(ll_ctx* ctx, LoopClosure* lc, const float4* full, int n, const int* d_n) {
  if (lc->done() || lc->stopped) return LL_OK;
  cudaStream_t s = ctx->stream;
  LoopInLayout il; LL_CUDA(ctx, lc->in.carve([&](Carve& k) { il.layout(k, lc->in_full, lc->in_scan); }));
  if (n > 0) LL_CUDA(ctx, cudaMemcpyAsync(il.full, full, (size_t)n * 16, cudaMemcpyDeviceToDevice, s));
  LL_CUDA(ctx, cudaMemcpyAsync(il.seg_end, d_n, sizeof(int), cudaMemcpyDeviceToDevice, s));   // one segment: the full cloud
  lc->seg.assign(1, 0); lc->seg_read = false; lc->piece = 0;
  return LL_OK;
}

size_t loop_step_capacity(const LoopClosure* lc) { return lc->in_scan; }   // loop_step_work transforms one step's cloud into `world` (in_scan points)

void loop_select_piece(LoopClosure* lc, int i) { lc->piece = i; }

namespace {

int loop_step_work(ll_ctx* ctx, LoopClosure* lc, const double* d_pose, bool pushed, int frame_index, const MapperWindow& mw) {
  cudaStream_t s = ctx->stream;
  const ll_loop_closure_cfg& c = lc->cfg;
  LoopInLayout il; LL_CUDA(ctx, lc->in.carve([&](Carve& k) { il.layout(k, lc->in_full, lc->in_scan); }));   // (reserved: no reallocation)
  // the step's pose: the mapper's, or after a correction C^-1 o the mapper's (loop closure stays in the odometry frame)
  ll_pose p; memcpy(p.q_wxyz, mw.q, sizeof(p.q_wxyz)); memcpy(p.t, mw.t, sizeof(p.t));
  if (lc->n_applied) {
    p = compose(inverse(lc->corr), p);
    double* h = ctx->pin->loop_pose; memcpy(h, p.q_wxyz, 4 * sizeof(double)); memcpy(h + 4, p.t, 3 * sizeof(double));
    FeedbackLayout fl; LL_CUDA(ctx, lc->fb.carve([&](Carve& k) { fl.layout(k, (size_t)std::max(lc->max_history, 0)); }));   // (reserved: no reallocation)
    LL_CUDA(ctx, cudaMemcpyAsync(fl.pose, h, 7 * sizeof(double), cudaMemcpyHostToDevice, s));
    d_pose = fl.pose;
  }
  if (!lc->seg_read) {   // the captured cloud's ends (the mapper step has synchronised the stream already: no wait here)
    LL_CUDA(ctx, cudaMemcpyAsync(lc->seg.data(), il.seg_end, lc->seg.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
    LL_CUDA(ctx, cudaStreamSynchronize(s));
    lc->seg_read = true;
  }
  const size_t off = lc->piece ? (size_t)lc->seg[lc->piece - 1] : 0;
  // the full cloud to the world frame (:1442), the full history (:1446-1459, :1480-1487)
  const int n = (int)((size_t)lc->seg[lc->piece] - off);
  float4* w = (float4*)lc->world.p;
  if (n > 0) LL_TRY(launch_transform(ctx, s, d_pose, il.full + off, n, w));
  if (pushed) LL_TRY(lc->his.push(ctx, w, (size_t)n));
  if ((int)lc->his.segs.size() > lc->max_history) lc->his.pop_front();
  // the full map and every open keyframe (:1527-1533)
  std::vector<ll_keyframe*> open(lc->open.size());
  for (size_t k = 0; k < open.size(); k++) open[k] = lc->open[k].kf;
  LL_TRY(ll_keyframe_append(ctx, lc->full, w, (size_t)n, LL_FMT_XYZI16, LL_DEVICE, open.data(), (int)open.size()));
  for (auto& o : lc->open) o.frames++;
  // close the front keyframe (:1534-1543)
  ll_keyframe* closing = nullptr;
  if (lc->open.front().frames >= c.scans_of_each_keyframe) { closing = lc->open.front().kf; lc->open.erase(lc->open.begin()); }
  // open a keyframe (:1545-1563): the history, down-sampled as :943-944 will filter it, is the back keyframe's accumulated cloud
  if (lc->open.back().frames >= c.scans_between_two_keyframe) {
    const size_t used = lc->acc_end.empty() ? 0 : lc->acc_end.back(), live = lc->his.live();
    LL_TRY(grow_keep(ctx, lc->acc, used * 16, (used + live) * 16 + 64));
    int kept = 0;
    if (live > 0) {
      int* d_cnt = (int*)((char*)lc->acc.p + lc->acc.cap - 64);
      LL_TRY(launch_voxel_grid(ctx, s, ctx->scratch, lc->his.data(), (int)live, nullptr, (float)c.surround_pointcloud_resolution, (float4*)lc->acc.p + used, d_cnt));
      LL_CUDA(ctx, cudaMemcpyAsync(&kept, d_cnt, sizeof(int), cudaMemcpyDeviceToHost, s));
      LL_CUDA(ctx, cudaStreamSynchronize(s));
    }
    lc->acc_end.push_back(used + (size_t)kept);
    lc->his.clear();
    ll_keyframe* kf = nullptr;
    LL_TRY(ll_keyframe_create(ctx, &kf));
    lc->open.push_back({kf, 0});
  }
  if (!closing) return LL_OK;
  // process it now (:931-960): analyze, the pose and its odometry edge, then the search
  lc->kfs.push_back(closing);
  lc->poses.push_back(p);
  lc->kf_frame.push_back(frame_index);
  const int id = (int)lc->kfs.size() - 1;
  if (id >= 1) { ll_pg_edge e; pg_odometry_edge(&lc->poses[id - 1], id - 1, &lc->poses[id], id, &e); lc->edges.push_back(e); }
  ll_keyframe_info info;
  LL_TRY(ll_keyframe_analyze(ctx, lc->full, closing, c.incremental_cov, &info));
  std::vector<int> cand(id + 1);
  int nc = 0;
  // the gap after the last loop (L its newest keyframe): a keyframe with id - L < min_keyframes_between_loops is recorded, not searched
  const bool search = lc->loops.empty() || id - std::max(lc->loops.back().id_begin, lc->loops.back().id_end) >= lc->policy.min_keyframes_between_loops;
  if (search) LL_TRY(ll_loop_search(ctx, lc->kfs.data(), id + 1, id, &c.loop, nullptr, nullptr, cand.data(), &nc));
  cand.resize(nc);
  ll_loop_event* ke = log_push(lc, LL_LOOP_KEYFRAME);
  ke->ending_frame_idx = frame_index; ke->n_candidates = nc; ke->info = info;
  memcpy(ke->q_wxyz, p.q_wxyz, sizeof(p.q_wxyz)); memcpy(ke->t, p.t, sizeof(p.t));
  return loop_align(ctx, lc, cand, mw);
}

}  // namespace

// Loop closure never fails the step: an error of its work other than LL_ERR_CUDA is logged (LL_LOOP_ERROR) and stops it for good.
int loop_step(ll_ctx* ctx, LoopClosure* lc, const double* d_pose, bool pushed, int frame_index, const MapperWindow& mw) {
  if (lc->done() || lc->stopped) return LL_OK;
  const int st = loop_step_work(ctx, lc, d_pose, pushed, frame_index, mw);
  if (st == LL_OK || st == LL_ERR_CUDA) return st;
  ll_loop_event* e = log_push(lc, LL_LOOP_ERROR);
  e->status = st; e->ending_frame_idx = frame_index;
  lc->stopped = true;   // (the context's last error names the failure)
  return LL_OK;
}

int loop_read(LoopClosure* lc, ll_loop_event* out, int cap, int* n, int* n_dropped) {
  if (lc) { lc->log.read(out, cap, n, n_dropped); return LL_OK; }
  *n = 0;
  if (n_dropped) *n_dropped = 0;
  return LL_OK;
}

int loop_result(const LoopClosure* lc, int* n, int* closed, ll_pose* poses_ori, ll_pose* poses_opt, int cap, ll_pg_edge* edge) {
  const int N = lc ? (int)lc->poses.size() : 0;
  const bool any = lc && !lc->loops.empty();
  if ((poses_ori || poses_opt) && cap < N) return LL_ERR_CAPACITY;
  if (n) *n = N;
  if (closed) *closed = any ? 1 : 0;
  if (poses_ori && N) memcpy(poses_ori, lc->poses.data(), N * sizeof(ll_pose));
  if (poses_opt && N) {   // the latest optimum for its n_opt keyframes, poses_ori after them
    const int n_opt = any ? (int)lc->opt.size() : 0;
    if (n_opt) memcpy(poses_opt, lc->opt.data(), n_opt * sizeof(ll_pose));
    if (N > n_opt) memcpy(poses_opt + n_opt, lc->poses.data() + n_opt, (N - n_opt) * sizeof(ll_pose));
  }
  if (edge) { if (any) *edge = lc->loops.back(); else memset(edge, 0, sizeof(*edge)); }
  return LL_OK;
}

int loop_edges(const LoopClosure* lc, ll_pg_edge* edges, int cap, int* n_loops) {
  const int n = lc ? (int)lc->loops.size() : 0;
  if (edges && cap < n) return LL_ERR_CAPACITY;
  *n_loops = n;
  if (edges && n) memcpy(edges, lc->loops.data(), n * sizeof(ll_pg_edge));
  return LL_OK;
}

// The pose graph of reserve_keyframes poses and reserve_keyframes - 1 + max_loops edges (every odometry edge and every loop edge), so that no
// solve up to reserve_keyframes allocates device memory.  Built aside: a failure changes nothing.
static int loop_reserve_graph(ll_ctx* ctx, LoopClosure* lc, int max_loops) {
  const int K = std::max(lc->cfg.reserve_keyframes, 2);
  ll_pose_graph* pg = nullptr;
  LL_TRY(ll_pose_graph_create(ctx, K, K - 1 + max_loops, &pg));
  ll_pose_graph_release(lc->pg);
  lc->pg = pg;
  return LL_OK;
}

int loop_set_policy(ll_ctx* ctx, LoopClosure* lc, const ll_loop_policy* p) {
  ll_loop_policy q{1, 0};
  if (p) q = *p;
  if (!lc) { ctx->set_error("loop closure is off: set it before its policy"); return LL_ERR_INVALID; }
  if (!lc->loops.empty()) { ctx->set_error("a loop has closed already: the policy is set before the first loop"); return LL_ERR_INVALID; }
  if (q.max_loops < 1 || q.max_loops > LL_MAX_LOOPS) { ctx->set_error("max_loops must be 1 ... LL_MAX_LOOPS"); return LL_ERR_INVALID; }
  if (q.min_keyframes_between_loops < 0) { ctx->set_error("min_keyframes_between_loops must be >= 0"); return LL_ERR_INVALID; }
  cudaSetDevice(ctx->device);
  if (q.max_loops != lc->policy.max_loops) LL_TRY(loop_reserve_graph(ctx, lc, q.max_loops));
  lc->policy = q;
  return LL_OK;
}

int loop_set_feedback(ll_ctx* ctx, LoopClosure* lc, const ll_mapper_config& mcfg, int on) {
  if (!lc) { ctx->set_error("loop closure is off: set it before loop feedback"); return LL_ERR_INVALID; }
  if (!lc->loops.empty()) { ctx->set_error("a loop has closed already: loop feedback is set before the first loop"); return LL_ERR_INVALID; }
  if (on && mcfg.matching_mode != 0) { ctx->set_error("loop feedback needs matching mode 0 (a cell-map point of mode 1 does not record its step)"); return LL_ERR_INVALID; }
  if (on && mcfg.maximum_history_size > LL_LOOP_FEEDBACK_MAX_SEGMENTS) { ctx->set_error("loop feedback: maximum_history_size above LL_LOOP_FEEDBACK_MAX_SEGMENTS"); return LL_ERR_INVALID; }
  if (on && std::any_of(lc->kf_frame.begin(), lc->kf_frame.end(), [](int f) { return f < 0; })) {
    ctx->set_error("loop feedback: keyframes restored from a loop image that does not record their frame indices"); return LL_ERR_INVALID;
  }
  if (on) LL_TRY(feedback_reserve(ctx, lc));
  lc->feedback = on != 0;
  return LL_OK;
}

void loop_correction(const LoopClosure* lc, double q_wxyz[4], double t[3], int* n_applied) {
  const ll_pose c = lc ? lc->corr : IDENTITY;
  memcpy(q_wxyz, c.q_wxyz, sizeof(c.q_wxyz)); memcpy(t, c.t, sizeof(c.t));
  if (n_applied) *n_applied = lc ? lc->n_applied : 0;
}

int loop_cloud(ll_ctx* ctx, const LoopClosure* lc, int k, ll_point* out_host, size_t cap, size_t* n_out, const ll_point** out_dev) {
  if (!lc || lc->loops.empty()) { ctx->set_error("no loop closed"); return LL_ERR_INVALID; }
  const int N = (int)lc->opt.size();   // n_opt: loop_refine's layout of the latest loop
  if (k < 0 || k >= N || (N - 1 - k) % 2 != 0) { ctx->set_error("keyframe k is not one the latest loop publishes (n_opt - 1, n_opt - 3, ...)"); return LL_ERR_INVALID; }
  RefineLayout rl; Carve c(lc->refine.p); rl.layout(c, lc->acc_end[N - 1]);
  // a chunk's outputs start where its inputs do (keyframes 256 c ...): keyframe k's output ends at ref_end[k] and starts at its predecessor's
  // end, or at the chunk's start
  const size_t o0 = k % 256 ? (size_t)lc->ref_end[k - 1] : (k ? lc->acc_end[k - 1] : 0), o1 = (size_t)lc->ref_end[k];
  *n_out = o1 - o0;
  const ll_point* d = *n_out ? (const ll_point*)(rl.out + o0) : nullptr;
  if (out_dev) *out_dev = d;
  if (out_host && *n_out) {
    cudaSetDevice(ctx->device);
    LL_CUDA(ctx, cudaMemcpyAsync(out_host, d, std::min(*n_out, cap) * 16, cudaMemcpyDeviceToHost, ctx->stream));
    LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  return LL_OK;
}

// ---------------------------------------------------------------------------------------------- loop image
// Format: include/loamlivox_b200.h ("loop image").  One host validator serves ll_loop_image_info and ll_mapper_loop_load, before anything
// touches the device; the save writes the sections back to back in index order.
namespace {

const ImageKind LOOP_IMAGE{LL_LOOP_IMAGE_MAGIC, "loop", LL_LOOP_IMAGE_VERSION, LL_LOOP_IMAGE_VERSION_FEEDBACK, sizeof(ll_loop_closure_cfg), "ll_loop_closure_cfg",
                           LL_LOOP_IMAGE_SECTIONS, LL_LOOP_IMAGE_VERSION_FEEDBACK};
const size_t LI_ACC_HEAD = 8, LI_IMG = 4 * 3600 * 4;                   // the accumulated section's fixed part; one keyframe's four images
const size_t LI_STAMP = offsetof(ll_loop_image_scalars, closed);       // the binding stamp: the scalars before `closed`
const size_t LI_LOOP2_HEAD = sizeof(ll_loop_policy) + 8;               // version 2's LOOP section: the policy, n_loops, 0
const size_t LI_FB_HEAD = 8 + sizeof(ll_pose) + 16;                    // version 3's FEEDBACK section: on, n_applied, C, n_keyframes, n_segments

bool policy_default(const ll_loop_policy& p) { return p.max_loops == 1 && p.min_keyframes_between_loops == 0; }
int edge_newest(const ll_pg_edge& e) { return std::max(e.id_begin, e.id_end); }

struct LoopView {   // a validated loop image
  ll_loop_image_header h; ll_image_section sec[LL_LOOP_IMAGE_SECTIONS_FEEDBACK]; ll_loop_closure_cfg cfg; ll_loop_image_scalars sc;
  CellsView cells;
  HistoryView his;
  const uint8_t* open = nullptr; const uint8_t* refs = nullptr; int64_t open_cells = 0;
  const uint8_t *infos = nullptr, *poses = nullptr, *edges = nullptr, *images = nullptr, *clouds = nullptr; int64_t cloud_pts = 0;
  int64_t n_acc = 0, acc_pts = 0; const uint8_t* acc_end = nullptr; const uint8_t* acc = nullptr;
  ll_loop_policy policy{1, 0}; int64_t n_loops = 0, n_opt = 0;   // the LOOP section: the policy (version 2), loop edges and optimized poses
  const uint8_t* loop_edges = nullptr; const uint8_t* loop_opt = nullptr; const uint8_t* events = nullptr;
  // the FEEDBACK section (version 3): n_applied, C, the keyframes' and the window segments' frame indices
  bool feedback = false; int n_applied = 0; ll_pose corr; int64_t n_fb_seg = 0; const uint8_t* kf_frame = nullptr; const uint8_t* seg_frame = nullptr;
};

bool finite_edge(const ll_pg_edge& e) { return finite_d(e.q_wxyz, 4) && finite_d(e.t, 3) && finite_d(e.information, 36); }

// LL_OK, or the code and what is wrong.  load: the image is to be loaded with cfg (NULL: the image's config), so the cell table that cfg's
// max_cells gives must hold its cells; ll_loop_image_info reports the cell count instead (an image saved by a mapper loaded with a larger
// max_cells can need one).
int loop_validate(const void* image, size_t bytes, bool load, const ll_loop_closure_cfg* cfg, LoopView* v, std::string* err) {
  auto fail = [&](const std::string& msg, int code = LL_ERR_INVALID) { if (err) *err = msg; return code; };
  LL_TRY(image_structure(image, bytes, LOOP_IMAGE, v->sec, err));
  const uint8_t* b = (const uint8_t*)image;
  memcpy(&v->h, b, sizeof(v->h));
  auto sec = [&](int k) { return b + v->sec[k].offset; };
  auto len = [&](int k) { return (uint64_t)v->sec[k].length; };
  // config: ll_mapper_set_loop_closure's checks
  if (len(LL_LOOP_IMAGE_CONFIG) != sizeof(ll_loop_closure_cfg)) return fail("config section length");
  memcpy(&v->cfg, sec(LL_LOOP_IMAGE_CONFIG), sizeof(v->cfg));
  if (const char* e = loop_cfg_error(v->cfg)) return fail(std::string("config: ") + e);
  { const ll_loop_closure_cfg z = loop_cfg_canonical(v->cfg); if (memcmp(&z, &v->cfg, sizeof(z)) != 0) return fail("config padding not zero"); }
  // scalars
  if (len(LL_LOOP_IMAGE_SCALARS) != sizeof(ll_loop_image_scalars)) return fail("scalars section length");
  memcpy(&v->sc, sec(LL_LOOP_IMAGE_SCALARS), sizeof(v->sc));
  const ll_loop_image_scalars& sc = v->sc;
  if (!std::isfinite(sc.last_time_stamp) || !finite_d(sc.q_w_curr, 4) || !finite_d(sc.t_w_curr, 3)) return fail("non-finite pose or time stamp");
  if (sc.frame_index < 0 || (sc.matching_mode != 0 && sc.matching_mode != 1) || sc.threshold_cell_revisit < 1 || !(sc.cell_resolution > 0.f) ||
      !std::isfinite(sc.cell_resolution) || sc.pieces < 1 || sc.pieces > LL_MAX_PIECES)
    return fail("binding stamp out of range");
  if ((sc.closed != 0 && sc.closed != 1) || (sc.stopped != 0 && sc.stopped != 1) || sc.n_keyframes < 0 || sc.n_open < 1 || sc.n_events < 0 ||
      sc.n_events > LL_LOOP_LOG || sc.n_dropped < 0)
    return fail("scalars out of range");
  const int64_t K = sc.n_keyframes;
  // the full map with its incarnation ordinals, and the full history
  if (const char* e = cells_section(sec(LL_LOOP_IMAGE_CELLS), len(LL_LOOP_IMAGE_CELLS), true, &v->cells)) return fail(e);
  if (const char* e = history_section(sec(LL_LOOP_IMAGE_HISTORY), len(LL_LOOP_IMAGE_HISTORY), false, &v->his)) return fail(e);
  if (sc.maximum_history_size >= 0 && v->his.n_seg > sc.maximum_history_size) return fail("more history segments than maximum_history_size");
  // open keyframes: their cells (cell rank, ordinal) strictly ascending and existing in the map
  {
    const uint8_t* p = sec(LL_LOOP_IMAGE_OPEN); const uint64_t L = len(LL_LOOP_IMAGE_OPEN);
    const uint64_t head = sizeof(ll_loop_image_open) * (uint64_t)sc.n_open;
    if (head > L) return fail("open-keyframe section shorter than its records");
    uint64_t refs = 0;
    for (int k = 0; k < sc.n_open; k++) {
      const ll_loop_image_open o = img_get<ll_loop_image_open>(p + sizeof(ll_loop_image_open) * k);
      if (o.frames < 0 || o.accumulate_frames < 0 || o.n_cells < 0 || (uint64_t)o.n_cells > L / 8) return fail("open keyframe out of range");
      if (o.accumulate_frames == 0 && o.n_cells > 0) return fail("open keyframe with cells but no append");
      refs += (uint64_t)o.n_cells;
    }
    if (head + sizeof(ll_loop_image_ref) * refs != L) return fail("open-keyframe cells disagree with the section length");
    const uint8_t* r = p + head;
    for (int k = 0; k < sc.n_open; k++) {
      const int64_t n = img_get<ll_loop_image_open>(p + sizeof(ll_loop_image_open) * k).n_cells;
      for (int64_t i = 0; i < n; i++, r += 8) {
        const ll_loop_image_ref x = img_get<ll_loop_image_ref>(r);
        if (x.cell < 0 || x.cell >= v->cells.n_cells || x.incarnation < 0 || x.incarnation > img_get<int32_t>(v->cells.cur + 4 * (int64_t)x.cell))
          return fail("open keyframe refers to a cell or incarnation the map does not hold");
        if (i > 0) {
          const ll_loop_image_ref y = img_get<ll_loop_image_ref>(r - 8);
          if (!(y.cell < x.cell || (y.cell == x.cell && y.incarnation < x.incarnation))) return fail("open keyframe's cells not strictly ascending");
        }
      }
    }
    v->open = p; v->refs = p + head; v->open_cells = (int64_t)refs;
  }
  // closed keyframes: infos, poses, the odometry edges between neighbours, images, typed clouds
  {
    if (len(LL_LOOP_IMAGE_KEYFRAMES) != sizeof(ll_keyframe_info) * (uint64_t)K || len(LL_LOOP_IMAGE_POSES) != sizeof(ll_pose) * (uint64_t)K ||
        len(LL_LOOP_IMAGE_EDGES) != sizeof(ll_pg_edge) * (uint64_t)(K ? K - 1 : 0) || len(LL_LOOP_IMAGE_IMAGES) != LI_IMG * (uint64_t)K)
      return fail("keyframe sections disagree with n_keyframes");
    v->infos = sec(LL_LOOP_IMAGE_KEYFRAMES); v->poses = sec(LL_LOOP_IMAGE_POSES); v->edges = sec(LL_LOOP_IMAGE_EDGES); v->images = sec(LL_LOOP_IMAGE_IMAGES);
    uint64_t cloud = 0;
    for (int64_t k = 0; k < K; k++) {
      const ll_keyframe_info in = img_get<ll_keyframe_info>(v->infos + sizeof(ll_keyframe_info) * k);
      if (in.cells < 0 || in.line_cells < 0 || in.plane_cells < 0 || (int64_t)in.line_cells + in.plane_cells > in.cells || in.accumulate_frames < 0 ||
          in.all_points > ((size_t)1 << 31) || in.line_points > in.all_points || in.plane_points > in.all_points - in.line_points)
        return fail("keyframe info out of range");
      if (in.cells == 0 && in.all_points != 0) return fail("keyframe info out of range");
      const float f[] = {in.center[0], in.center[1], in.center[2], in.roi_range, in.ratio_nonzero_line, in.ratio_nonzero_plane};
      for (float x : f) if (!std::isfinite(x)) return fail("non-finite keyframe info");
      if (!finite_pose(img_get<ll_pose>(v->poses + sizeof(ll_pose) * k))) return fail("non-finite keyframe pose");
      if (k > 0) {
        const ll_pg_edge e = img_get<ll_pg_edge>(v->edges + sizeof(ll_pg_edge) * (k - 1));
        if (e.id_begin != k - 1 || e.id_end != k || !finite_edge(e)) return fail("odometry edge out of range");
      }
      const uint8_t* im = v->images + LI_IMG * k;
      for (size_t q = 0; q < LI_IMG / 4; q++) if (!std::isfinite(img_get<float>(im + 4 * q))) return fail("non-finite keyframe image");
      cloud += in.line_points + in.plane_points;
    }
    if (len(LL_LOOP_IMAGE_CLOUDS) != 16 * cloud) return fail("keyframe clouds disagree with the infos");
    v->clouds = sec(LL_LOOP_IMAGE_CLOUDS); v->cloud_pts = (int64_t)cloud;
    for (uint64_t q = 0; q < cloud; q++) if (!finite_xyz(v->clouds + 16 * q)) return fail("non-finite keyframe cloud point");
  }
  // accumulated clouds: one per closed keyframe and per open one but the newest
  {
    const uint8_t* p = sec(LL_LOOP_IMAGE_ACCUMULATED); const uint64_t L = len(LL_LOOP_IMAGE_ACCUMULATED);
    if (L < LI_ACC_HEAD) return fail("accumulated section shorter than its count");
    const int64_t n = img_get<int64_t>(p);
    if (n != K + sc.n_open - 1) return fail("accumulated clouds != closed + open keyframes - 1");
    if ((uint64_t)n > (L - LI_ACC_HEAD) / 8) return fail("accumulated counts disagree with the section length");
    int64_t prev = 0;
    for (int64_t k = 0; k < n; k++) {
      const int64_t e = img_get<int64_t>(p + LI_ACC_HEAD + 8 * k);
      if (e < prev) return fail("accumulated cloud ends decreasing");
      prev = e;
    }
    if (prev > INT32_MAX || LI_ACC_HEAD + 8 * (uint64_t)n + 16 * (uint64_t)prev != L) return fail("accumulated counts disagree with the section length");
    v->n_acc = n; v->acc_pts = prev; v->acc_end = p + LI_ACC_HEAD; v->acc = p + LI_ACC_HEAD + 8 * n;
    for (int64_t k = 0; k < prev; k++) if (!finite_xyz(v->acc + 16 * k)) return fail("non-finite accumulated point");
  }
  // the loop.  Version 1: the edge between two keyframes and the optimized poses, only when closed.  Versions 2 and 3: the policy, the loop
  // edges in closing order and the latest optimized poses
  {
    const uint64_t L = len(LL_LOOP_IMAGE_LOOP);
    const uint8_t* p = sec(LL_LOOP_IMAGE_LOOP);
    if (v->h.version == LL_LOOP_IMAGE_VERSION) {
      if (!sc.closed) { if (L != 0) return fail("loop section of an unclosed image not empty"); }
      else {
        if (K < 2) return fail("a closed loop needs two keyframes");
        if (L != sizeof(ll_pg_edge) + sizeof(ll_pose) * (uint64_t)K) return fail("loop section disagrees with n_keyframes");
        const ll_pg_edge e = img_get<ll_pg_edge>(p);
        if (e.id_begin < 0 || e.id_begin >= K || e.id_end < 0 || e.id_end >= K || !finite_edge(e)) return fail("loop edge out of range");
        v->n_loops = 1; v->n_opt = K;
      }
    } else {
      if (L < LI_LOOP2_HEAD) return fail("version-2 loop section shorter than its policy and count");
      v->policy = img_get<ll_loop_policy>(p);
      const int32_t nl = img_get<int32_t>(p + sizeof(ll_loop_policy)), pad = img_get<int32_t>(p + sizeof(ll_loop_policy) + 4);
      const int lo = v->h.version == LL_LOOP_IMAGE_VERSION_POLICY ? 2 : 1;   // (without feedback the default policy writes version 1)
      if (v->policy.max_loops < lo || v->policy.max_loops > LL_MAX_LOOPS) return fail("max_loops outside " + std::to_string(lo) + " ... LL_MAX_LOOPS");
      if (v->policy.min_keyframes_between_loops < 0) return fail("negative min_keyframes_between_loops");
      if (pad != 0) return fail("loop section padding not zero");
      if (nl < 0 || nl > v->policy.max_loops) return fail("n_loops outside 0 ... max_loops");
      if (L < LI_LOOP2_HEAD + sizeof(ll_pg_edge) * (uint64_t)nl) return fail("loop section shorter than its edges");
      int prev = -1;
      for (int k = 0; k < nl; k++) {
        const ll_pg_edge e = img_get<ll_pg_edge>(p + LI_LOOP2_HEAD + sizeof(ll_pg_edge) * k);
        if (e.id_begin < 0 || e.id_begin >= K || e.id_end < 0 || e.id_end >= K || e.id_begin == e.id_end || !finite_edge(e)) return fail("loop edge out of range");
        const int nw = edge_newest(e);
        if (k > 0 && (nw <= prev || nw - prev < v->policy.min_keyframes_between_loops)) return fail("loop edges' newest keyframes not increasing by the gap");
        prev = nw;
      }
      v->n_loops = nl; v->n_opt = nl ? prev + 1 : 0;
      if ((sc.closed != 0) != (nl > 0)) return fail("closed disagrees with n_loops");
      if (L != LI_LOOP2_HEAD + sizeof(ll_pg_edge) * (uint64_t)nl + sizeof(ll_pose) * (uint64_t)v->n_opt) return fail("loop section disagrees with its edges");
    }
    const size_t head = v->h.version == LL_LOOP_IMAGE_VERSION ? 0 : LI_LOOP2_HEAD;
    v->loop_edges = p + head;
    v->loop_opt = p + head + sizeof(ll_pg_edge) * (size_t)v->n_loops;
    for (int64_t k = 0; k < v->n_opt; k++) if (!finite_pose(img_get<ll_pose>(v->loop_opt + sizeof(ll_pose) * k))) return fail("non-finite optimized pose");
  }
  // loop feedback (version 3): the correction, the keyframes' frame indices and the window segments' (their count is checked by the load)
  if (v->h.version == LL_LOOP_IMAGE_VERSION_FEEDBACK) {
    const uint8_t* p = sec(LL_LOOP_IMAGE_FEEDBACK); const uint64_t L = len(LL_LOOP_IMAGE_FEEDBACK);
    if (L < LI_FB_HEAD) return fail("feedback section shorter than its head");
    const int32_t on = img_get<int32_t>(p), na = img_get<int32_t>(p + 4);
    v->corr = img_get<ll_pose>(p + 8);
    const int64_t nk = img_get<int64_t>(p + 8 + sizeof(ll_pose)), ns = img_get<int64_t>(p + 16 + sizeof(ll_pose));
    if (on != 1) return fail("feedback flag not 1");
    if (na < 0 || na > v->n_loops || (na < v->n_loops && !sc.stopped)) return fail("corrections applied outside 0 ... n_loops (fewer only when stopped)");
    if (!finite_pose(v->corr)) return fail("non-finite correction");
    if (na == 0 && memcmp(&v->corr, &IDENTITY, sizeof(ll_pose)) != 0) return fail("a correction other than the identity before one was applied");
    if (nk != K) return fail("feedback keyframes disagree with n_keyframes");
    if (ns < 0 || (uint64_t)ns > (L - LI_FB_HEAD) / 4 || LI_FB_HEAD + 4 * ((uint64_t)nk + (uint64_t)ns) != L) return fail("feedback counts disagree with the section length");
    if (sc.maximum_history_size >= 0 && ns > sc.maximum_history_size) return fail("more window segments than maximum_history_size");
    const uint8_t* kf = p + LI_FB_HEAD; const uint8_t* sg = kf + 4 * nk;
    for (int64_t k = 0; k < nk; k++) {
      const int32_t f = img_get<int32_t>(kf + 4 * k);
      if (f < 0 || f > sc.frame_index || (k && f <= img_get<int32_t>(kf + 4 * (k - 1)))) return fail("keyframe frame indices not strictly ascending within 0 ... frame_index");
    }
    for (int64_t k = 0; k < ns; k++) {
      const int32_t f = img_get<int32_t>(sg + 4 * k);
      if (f < 0 || f > sc.frame_index || (k && f <= img_get<int32_t>(sg + 4 * (k - 1)))) return fail("window frame indices not strictly ascending within 0 ... frame_index");
    }
    v->feedback = true; v->n_applied = na; v->n_fb_seg = ns; v->kf_frame = kf; v->seg_frame = sg;
  }
  // the unread events
  {
    if (len(LL_LOOP_IMAGE_EVENTS) != sizeof(ll_loop_event) * (uint64_t)sc.n_events) return fail("events disagree with n_events");
    v->events = sec(LL_LOOP_IMAGE_EVENTS);
    for (int k = 0; k < sc.n_events; k++) {
      const ll_loop_event e = img_get<ll_loop_event>(v->events + sizeof(ll_loop_event) * k);
      if (e.kind < LL_LOOP_KEYFRAME || e.kind > LL_LOOP_ERROR) return fail("unknown event kind");
      if (e.summary.cycles_eval || e.summary.cycles_elim || e.summary.cycles_border || e.summary.cycles_total) return fail("event with timing counters not zero");
    }
  }
  // the caller's config: the image's but for the allocation sizes
  if (cfg) {
    ll_loop_closure_cfg x = loop_cfg_canonical(*cfg);
    x.max_cells = v->cfg.max_cells; x.reserve_map_points = v->cfg.reserve_map_points; x.reserve_history_points = v->cfg.reserve_history_points;
    x.reserve_keyframes = v->cfg.reserve_keyframes;
    if (memcmp(&x, &v->cfg, sizeof(x)) != 0) return fail("cfg differs from the image's config in a field other than max_cells and reserve_*");
    if (const char* e = loop_cfg_error(*cfg)) return fail(std::string("cfg: ") + e);
  }
  const int max_cells = cfg ? cfg->max_cells : v->cfg.max_cells;
  if (const char* e = load_capacity(v->cells, v->his, load ? &max_cells : nullptr)) return fail(e, LL_ERR_CAPACITY);
  return LL_OK;
}

// The loop-closure state of a validated image into lc, just made by loop_set (its first open keyframe released) over the mapper it binds to.
int loop_restore(ll_ctx* ctx, LoopClosure* lc, const LoopView& v) {
  cudaStream_t s = ctx->stream;
  const ll_loop_image_scalars& sc = v.sc;
  const int K = sc.n_keyframes;
  // the full map, its epochs the image's ordinals, and the full history
  std::vector<int> slot(v.cells.n_cells);
  LL_TRY(cells_restore(ctx, lc->full, v.cells, true, slot.data()));
  LL_TRY(history_restore(ctx, lc->his, v.his));
  // open keyframes: (cell rank, ordinal) back to (slot, epoch) of the new table
  const uint8_t* r = v.refs;
  for (int k = 0; k < sc.n_open; k++) {
    const ll_loop_image_open o = img_get<ll_loop_image_open>(v.open + sizeof(ll_loop_image_open) * k);
    std::vector<unsigned long long> keys(o.n_cells), ids(o.n_cells);
    for (int64_t i = 0; i < o.n_cells; i++, r += 8) {
      const ll_loop_image_ref x = img_get<ll_loop_image_ref>(r);
      keys[i] = img_get<ll_image_cell>(v.cells.rec + 16 * (int64_t)x.cell).key;
      ids[i] = ((unsigned long long)(unsigned)slot[x.cell] << 32) | (unsigned)x.incarnation;
    }
    ll_keyframe* kf = nullptr;
    LL_TRY(ll_keyframe_create(ctx, &kf));
    lc->open.push_back({kf, o.frames});
    LL_TRY(kf_restore_open(ctx, lc->full, kf, keys.data(), ids.data(), (int)o.n_cells, (unsigned)o.accumulate_frames));
  }
  // closed keyframes, their poses and odometry edges
  size_t cloud = 0;
  for (int k = 0; k < K; k++) {
    const ll_keyframe_info in = img_get<ll_keyframe_info>(v.infos + sizeof(ll_keyframe_info) * k);
    ll_keyframe* kf = nullptr;
    LL_TRY(ll_keyframe_create(ctx, &kf));
    lc->kfs.push_back(kf);
    LL_TRY(kf_restore_closed(ctx, lc->full, kf, in, (const float*)(v.images + LI_IMG * k), v.clouds + 16 * cloud));
    cloud += in.line_points + in.plane_points;
    lc->poses.push_back(img_get<ll_pose>(v.poses + sizeof(ll_pose) * k));
    if (k > 0) lc->edges.push_back(img_get<ll_pg_edge>(v.edges + sizeof(ll_pg_edge) * (k - 1)));
  }
  // accumulated clouds
  for (int64_t k = 0; k < v.n_acc; k++) lc->acc_end.push_back((size_t)img_get<int64_t>(v.acc_end + 8 * k));
  LL_TRY(grow_keep(ctx, lc->acc, 0, (size_t)v.acc_pts * 16 + 64));
  if (v.acc_pts) LL_CUDA(ctx, cudaMemcpyAsync(lc->acc.p, v.acc, (size_t)v.acc_pts * 16, cudaMemcpyHostToDevice, s));
  // the policy, the loops and the latest loop's refined clouds, recomputed
  if (!policy_default(v.policy)) LL_TRY(loop_set_policy(ctx, lc, &v.policy));
  lc->stopped = sc.stopped != 0;
  for (int64_t k = 0; k < v.n_loops; k++) lc->loops.push_back(img_get<ll_pg_edge>(v.loop_edges + sizeof(ll_pg_edge) * k));
  lc->opt.resize((size_t)v.n_opt);
  for (int64_t k = 0; k < v.n_opt; k++) lc->opt[k] = img_get<ll_pose>(v.loop_opt + sizeof(ll_pose) * k);
  if (v.n_loops) LL_TRY(loop_refine(ctx, lc));
  // loop feedback: on with its frame indices (version 3), else off with the keyframes' frame indices unknown
  lc->kf_frame.assign((size_t)K, -1);
  if (v.feedback) {
    LL_TRY(feedback_reserve(ctx, lc));
    lc->feedback = true;
    for (int k = 0; k < K; k++) lc->kf_frame[k] = img_get<int32_t>(v.kf_frame + 4 * k);
    lc->corr = v.corr; lc->n_applied = v.n_applied;
  }
  lc->log.restore(v.events, (size_t)sc.n_events, sc.n_dropped);   // the unread events
  LL_CUDA(ctx, cudaGetLastError());
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  return LL_OK;
}

}  // namespace

int loop_save(ll_ctx* ctx, const LoopClosure* lc, const ll_loop_image_scalars& stamp, const MapperWindow& mw, void* image, size_t cap, size_t* bytes) {
  cudaStream_t s = ctx->stream;
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  // the incarnations the open keyframes hold (sorted, distinct), on the device for the export
  std::vector<std::vector<unsigned long long>> okeys(lc->open.size()), oids(lc->open.size());
  std::vector<unsigned long long> held;
  uint64_t open_cells = 0;
  for (size_t k = 0; k < lc->open.size(); k++) {
    const int c = kf_cell_count(lc->open[k].kf);
    okeys[k].resize(c); oids[k].resize(c);
    LL_TRY(kf_cell_ids(ctx, lc->open[k].kf, okeys[k].data(), oids[k].data()));
    held.insert(held.end(), oids[k].begin(), oids[k].end());
    open_cells += c;
  }
  std::sort(held.begin(), held.end()); held.erase(std::unique(held.begin(), held.end()), held.end());
  struct Owned { DevBuf b; ~Owned() { b.release(); } } d_held;
  if (!held.empty()) {
    LL_CUDA(ctx, d_held.b.reserve(held.size() * 8));
    LL_CUDA(ctx, cudaMemcpyAsync(d_held.b.p, held.data(), held.size() * 8, cudaMemcpyHostToDevice, s));
  }
  const CmHeld H{(const unsigned long long*)d_held.b.p, (int)held.size()};
  CellsView cells; int nc = 0, live = 0, kept = 0;
  LL_TRY(cm_count(ctx, lc->full, &nc, &live, &cells.frame_idx, &cells.n_oor));
  LL_TRY(cm_count_kept(ctx, lc->full, H, &kept));
  cells.n_cells = nc; cells.n_pts = kept;
  const size_t K = lc->kfs.size();
  std::vector<ll_keyframe_info> infos(K);
  uint64_t cloud_pts = 0;
  for (size_t k = 0; k < K; k++) {
    if (ll_keyframe_get_info(lc->kfs[k], &infos[k]) != LL_OK) {   // only a keyframe whose analysis failed (LL_LOOP_ERROR) has none
      ctx->set_error("keyframe " + std::to_string(k) + " was closed by a loop closure that an error stopped and has no analysis: it cannot be saved");
      return LL_ERR_INVALID;
    }
    cloud_pts += infos[k].line_points + infos[k].plane_points;
  }
  const uint64_t acc_pts = lc->acc_end.empty() ? 0 : lc->acc_end.back();
  // v2: a policy other than the default (version 2) or loop feedback (version 3, which adds the FEEDBACK section); n_opt: the latest
  // optimization's keyframes
  const bool v3 = lc->feedback, v2 = v3 || !policy_default(lc->policy);
  const uint64_t n_seg = v3 ? mw.frame->size() : 0;
  const uint64_t n_loops = lc->loops.size(), n_opt = n_loops ? lc->opt.size() : 0;
  const uint64_t loop_len = v2 ? LI_LOOP2_HEAD + sizeof(ll_pg_edge) * n_loops + sizeof(ll_pose) * n_opt : n_loops ? sizeof(ll_pg_edge) + sizeof(ll_pose) * n_opt : 0;
  const uint64_t len[LL_LOOP_IMAGE_SECTIONS_FEEDBACK] = {
      sizeof(ll_loop_closure_cfg), sizeof(ll_loop_image_scalars), cells_bytes(cells, true), history_bytes(lc->his),
      sizeof(ll_loop_image_open) * lc->open.size() + sizeof(ll_loop_image_ref) * open_cells, sizeof(ll_keyframe_info) * K, sizeof(ll_pose) * K,
      sizeof(ll_pg_edge) * (K ? K - 1 : 0), LI_IMG * K, 16 * cloud_pts, LI_ACC_HEAD + 8 * lc->acc_end.size() + 16 * acc_pts, loop_len,
      sizeof(ll_loop_event) * lc->log.count, LI_FB_HEAD + 4 * (K + n_seg)};
  uint8_t hbuf[24 + 16 * LL_LOOP_IMAGE_SECTIONS_FEEDBACK];
  const uint32_t version = v3 ? LL_LOOP_IMAGE_VERSION_FEEDBACK : v2 ? LL_LOOP_IMAGE_VERSION_POLICY : LL_LOOP_IMAGE_VERSION;
  const size_t total = image_header(LOOP_IMAGE, version, len, hbuf);
  const size_t head = 24 + 16 * (size_t)LOOP_IMAGE.count(version);
  ll_image_section sec[LL_LOOP_IMAGE_SECTIONS_FEEDBACK];
  memcpy(sec, hbuf + 24, head - 24);
  *bytes = total;
  if (!image) return LL_OK;
  if (cap < total) { ctx->set_error("image buffer smaller than the loop image (query the size with image = NULL)"); return LL_ERR_CAPACITY; }
  uint8_t* b = (uint8_t*)image;
  auto at = [&](int k) { return b + sec[k].offset; };
  memcpy(b, hbuf, head);
  memcpy(at(LL_LOOP_IMAGE_CONFIG), &lc->cfg, sizeof(lc->cfg));
  ll_loop_image_scalars sc = stamp;
  sc.closed = lc->loops.empty() ? 0 : 1; sc.stopped = lc->stopped ? 1 : 0;
  sc.n_keyframes = (int32_t)K; sc.n_open = (int32_t)lc->open.size(); sc.n_events = (int32_t)lc->log.count; sc.n_dropped = lc->log.dropped;
  memcpy(at(LL_LOOP_IMAGE_SCALARS), &sc, sizeof(sc));
  // the full map with the held incarnations, the full history
  LL_TRY(cells_write(ctx, lc->full, cells, at(LL_LOOP_IMAGE_CELLS), &H));
  const uint8_t* ecells = at(LL_LOOP_IMAGE_CELLS) + CELLS_HEAD;
  LL_TRY(history_write(ctx, lc->his, at(LL_LOOP_IMAGE_HISTORY)));
  // open keyframes: (slot, epoch) as (cell rank by key, ordinal)
  uint8_t* p = at(LL_LOOP_IMAGE_OPEN);
  uint8_t* refs = p + sizeof(ll_loop_image_open) * lc->open.size();
  for (size_t k = 0; k < lc->open.size(); k++) {
    ll_loop_image_open o; memset(&o, 0, sizeof(o));
    o.frames = lc->open[k].frames; o.accumulate_frames = (int32_t)kf_accumulate_frames(lc->open[k].kf); o.n_cells = (int64_t)okeys[k].size();
    img_put(p + sizeof(o) * k, o);
    for (size_t i = 0; i < okeys[k].size(); i++, refs += 8) {
      int lo = 0, hi = (int)cells.n_cells;   // the cell's rank: its key in the exported list
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (img_get<ll_image_cell>(ecells + 16 * (size_t)mid).key < okeys[k][i]) lo = mid + 1; else hi = mid; }
      ll_loop_image_ref x; x.cell = lo;
      x.incarnation = cm_ordinal(held.data(), (int)held.size(), (int)(oids[k][i] >> 32), (int)(unsigned)(oids[k][i] & 0xffffffffull));
      img_put(refs, x);
    }
  }
  // closed keyframes
  size_t cloud = 0;
  uint8_t* clouds = at(LL_LOOP_IMAGE_CLOUDS);
  for (size_t k = 0; k < K; k++) {
    img_put(at(LL_LOOP_IMAGE_KEYFRAMES) + sizeof(ll_keyframe_info) * k, infos[k]);
    img_put(at(LL_LOOP_IMAGE_POSES) + sizeof(ll_pose) * k, lc->poses[k]);
    if (k > 0) img_put(at(LL_LOOP_IMAGE_EDGES) + sizeof(ll_pg_edge) * (k - 1), lc->edges[k - 1]);
    float* im = (float*)(at(LL_LOOP_IMAGE_IMAGES) + LI_IMG * k);
    LL_TRY(ll_keyframe_images(ctx, lc->kfs[k], im, im + 3600, im + 2 * 3600, im + 3 * 3600));
    size_t nl = 0, np = 0;
    LL_TRY(ll_keyframe_cloud(ctx, lc->kfs[k], LL_CELL_LINE, (ll_point*)(clouds + 16 * cloud), infos[k].line_points, &nl, nullptr));
    LL_TRY(ll_keyframe_cloud(ctx, lc->kfs[k], LL_CELL_PLANE, (ll_point*)(clouds + 16 * (cloud + nl)), infos[k].plane_points, &np, nullptr));
    cloud += nl + np;
  }
  // accumulated clouds
  p = at(LL_LOOP_IMAGE_ACCUMULATED);
  img_put<int64_t>(p, (int64_t)lc->acc_end.size());
  for (size_t k = 0; k < lc->acc_end.size(); k++) img_put<int64_t>(p + LI_ACC_HEAD + 8 * k, (int64_t)lc->acc_end[k]);
  if (acc_pts) LL_CUDA(ctx, cudaMemcpyAsync(p + LI_ACC_HEAD + 8 * lc->acc_end.size(), lc->acc.p, (size_t)acc_pts * 16, cudaMemcpyDeviceToHost, s));
  // the loop: version 1 the edge of the one loop, version 2 the policy and every loop edge; then the optimized poses
  p = at(LL_LOOP_IMAGE_LOOP);
  if (v2) {
    img_put(p, lc->policy); img_put<int32_t>(p + sizeof(ll_loop_policy), (int32_t)n_loops); img_put<int32_t>(p + sizeof(ll_loop_policy) + 4, 0);
    p += LI_LOOP2_HEAD;
  }
  if (n_loops) {
    memcpy(p, lc->loops.data(), sizeof(ll_pg_edge) * lc->loops.size());
    memcpy(p + sizeof(ll_pg_edge) * lc->loops.size(), lc->opt.data(), sizeof(ll_pose) * (size_t)n_opt);
  }
  // the unread events, oldest first
  for (size_t k = 0; k < lc->log.count; k++) {   // the pose graph's SM clock counters time the solve: not state, saved as 0
    ll_loop_event e = lc->log.at(k);
    e.summary.cycles_eval = e.summary.cycles_elim = e.summary.cycles_border = e.summary.cycles_total = 0;
    img_put(at(LL_LOOP_IMAGE_EVENTS) + sizeof(ll_loop_event) * k, e);
  }
  // loop feedback: the correction, then the keyframes' and the window segments' frame indices
  if (v3) {
    p = at(LL_LOOP_IMAGE_FEEDBACK);
    img_put<int32_t>(p, 1); img_put<int32_t>(p + 4, lc->n_applied); img_put(p + 8, lc->corr);
    img_put<int64_t>(p + 8 + sizeof(ll_pose), (int64_t)K); img_put<int64_t>(p + 16 + sizeof(ll_pose), (int64_t)n_seg);
    p += LI_FB_HEAD;
    for (size_t k = 0; k < K; k++, p += 4) img_put<int32_t>(p, lc->kf_frame[k]);
    for (uint64_t k = 0; k < n_seg; k++, p += 4) img_put<int32_t>(p, (*mw.frame)[k]);
  }
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  return LL_OK;
}

int loop_load(ll_ctx* ctx, LoopClosure** plc, const void* image, size_t bytes, const ll_loop_closure_cfg* cfg, const ll_loop_image_scalars& stamp,
              const ll_mapper_config& mcfg, int pieces, const MapperWindow& mw) {
  LoopView v; std::string err;
  const int st = loop_validate(image, bytes, true, cfg, &v, &err);
  if (st != LL_OK) { ctx->set_error("loop image refused: " + err); return st; }
  if (memcmp(&v.sc, &stamp, LI_STAMP) != 0) {
    ctx->set_error("loop image refused: its binding stamp (frame index, pose, time stamp, matching mode, cell_resolution, threshold_cell_revisit, "
                   "maximum_history_size, pieces) differs from the mapper's");
    return LL_ERR_INVALID;
  }
  if (v.feedback && ((size_t)v.n_fb_seg != mw.his[0]->segs.size() || (size_t)v.n_fb_seg != mw.his[1]->segs.size())) {
    ctx->set_error("loop image refused: its window segments differ from the mapper's history windows");
    return LL_ERR_INVALID;
  }
  if (v.feedback && mcfg.matching_mode != 0) { ctx->set_error("loop image refused: loop feedback needs matching mode 0"); return LL_ERR_INVALID; }
  cudaSetDevice(ctx->device);
  LoopClosure* lc = nullptr;
  LL_TRY(loop_set(ctx, &lc, cfg ? cfg : &v.cfg, mcfg, pieces));
  free_keyframes(lc);
  const int rs = loop_restore(ctx, lc, v);
  if (rs != LL_OK) { loop_release(lc); return rs; }
  lc->cfg = v.cfg;   // cfg's allocation sizes were read by loop_set only; later images keep the image's config
  if (v.feedback) mw.frame->clear();
  for (int64_t k = 0; v.feedback && k < v.n_fb_seg; k++) mw.frame->push_back(img_get<int32_t>(v.seg_frame + 4 * k));
  loop_release(*plc);
  *plc = lc;
  return LL_OK;
}

int loop_image_info(const void* image, size_t bytes, ll_loop_image_summary* info) {
  LoopView v;
  LL_TRY(loop_validate(image, bytes, false, nullptr, &v, nullptr));
  memset(info, 0, sizeof(*info));
  info->bytes = bytes; info->version = v.h.version;
  info->cells = v.cells.n_cells; info->cell_points = v.cells.n_pts; info->replaced_points = v.cells.replaced;
  info->history_points = v.his.n_pts; info->cloud_points = v.cloud_pts; info->accumulated_points = v.acc_pts;
  info->frame_index = v.sc.frame_index; info->matching_mode = v.sc.matching_mode; info->closed = v.sc.closed; info->stopped = v.sc.stopped;
  info->keyframes = v.sc.n_keyframes; info->open_keyframes = v.sc.n_open; info->events = v.sc.n_events; info->dropped = v.sc.n_dropped;
  info->max_incarnation = v.cells.max_cur;
  return LL_OK;
}

extern "C" int ll_loop_correction(const ll_pose* ori, const ll_pose* opt, const int* f, int n, int s, double q_wxyz[4], double t[3]) {
  if (!ori || !opt || !f || n < 1 || !q_wxyz || !t) return LL_ERR_INVALID;
  for (int k = 1; k < n; k++) if (f[k] <= f[k - 1]) return LL_ERR_INVALID;
  const ll_pose c = correction_at(ori, opt, f, n, s);
  memcpy(q_wxyz, c.q_wxyz, sizeof(c.q_wxyz)); memcpy(t, c.t, sizeof(c.t));
  return LL_OK;
}
