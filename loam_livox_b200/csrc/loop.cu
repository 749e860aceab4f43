// Loop closure inside the streaming mapper (ll_mapper_set_loop_closure; DESIGN.md §4.6): Laser_mapping::process_new_scan's keyframe block
// (loam_livox/source/laser_mapping.hpp:1442, 1446-1459, 1480-1487, 1523-1564) and service_loop_detection (:874-1127), run by the mapper step
// that appends its features, with every full cloud on the device.  Everything below is host orchestration of the library's own entry points
// (transform, VoxelGrid, ll_keyframe_*, ll_loop_search, ll_scene_align, the pose graph, the re-pose) plus one gather kernel.
#include <algorithm>
#include <cmath>
#include <cstring>
#include "common.cuh"
#include "kernels.cuh"

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
  bool closed = false;                               // if_end
  bool stopped = false;                              // an error of the loop work stopped it (LL_LOOP_ERROR)
  bool seg_read = false;                             // seg holds the captured cloud's ends (read by the first step after a capture)
  int piece = 0;                                     // the step's piece of the captured frame
  ll_pg_edge loop_edge{}; std::vector<ll_pose> opt;  // constrain_vec_temp.back(), temp_pose_3d_map
  DevBuf refine; std::vector<int> ref_end;           // RefineLayout: the re-posed clouds of every keyframe
  std::vector<ll_loop_event> ring; size_t first = 0, count = 0; int dropped = 0;
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
  if (c.max_cells < 0) return "max_cells must be >= 0";
  if (c.reserve_map_points < 0 || c.reserve_map_points > INT32_MAX || c.reserve_history_points < 0 || c.reserve_history_points > INT32_MAX)
    return "reservations must be 0 ... 2^31 - 1 points";
  if (c.reserve_keyframes < 0 || c.reserve_keyframes > (1 << 20)) return "reserve_keyframes must be 0 ... 2^20";
  return nullptr;
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

ll_loop_event* log_push(LoopClosure* lc, int kind) {
  if (lc->count == lc->ring.size()) { lc->first = (lc->first + 1) % lc->ring.size(); lc->count--; lc->dropped++; }
  ll_loop_event* e = &lc->ring[(lc->first + lc->count) % lc->ring.size()]; lc->count++;
  memset(e, 0, sizeof(*e)); e->kind = kind; e->keyframe = (int)lc->kfs.size() - 1;
  return e;
}

void free_keyframes(LoopClosure* lc) {
  for (auto& o : lc->open) ll_keyframe_release(o.kf);
  for (ll_keyframe* k : lc->kfs) ll_keyframe_release(k);
  lc->open.clear(); lc->kfs.clear();
}

// The candidates of the newest keyframe (ll_loop_search's, his ascending) through the alignment with the skips of :1048-1052 and
// :1113-1116, and on a loop the graph and the refined clouds (:1056-1100).
int loop_align(ll_ctx* ctx, LoopClosure* lc, const std::vector<int>& cand) {
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
    // the loop (:1056-1100): the edge, the graph on the odometry edges plus this one, the refined clouds
    ll_pose_graph_loop_edge(r.q_w_curr, r.t_w_curr, &lc->poses[his], his, &lc->poses[newest], newest, &lc->loop_edge);
    std::vector<ll_pg_edge> edges = lc->edges; edges.push_back(lc->loop_edge);
    lc->opt = lc->poses;
    ll_pg_summary sum;
    LL_TRY(ll_pose_graph_optimize(lc->pg, lc->opt.data(), n, edges.data(), (int)edges.size(), 200, &sum));
    // Mapping_refine::refine_pointcloud (if_save 0) of every keyframe, 256 per launch chain; the readers give the published ones
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
    ll_loop_event* ce = log_push(lc, LL_LOOP_CLOSED);
    ce->his = his; ce->edge = lc->loop_edge; ce->summary = sum;
    lc->closed = true;
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
  lc->cfg = *cfg; lc->cell_res = mcfg.cell_resolution; lc->revisit = mcfg.threshold_cell_revisit; lc->max_history = mcfg.maximum_history_size;
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
    lc->ring.resize(LL_LOOP_LOG);
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
  if (lc->closed || lc->stopped) return LL_OK;
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
  if (lc->closed || lc->stopped) return LL_OK;
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
  if (lc->closed || lc->stopped) return LL_OK;
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

int loop_step_work(ll_ctx* ctx, LoopClosure* lc, const double* d_pose, bool pushed, int frame_index, const double q_w_curr[4], const double t_w_curr[3]) {
  cudaStream_t s = ctx->stream;
  const ll_loop_closure_cfg& c = lc->cfg;
  LoopInLayout il; LL_CUDA(ctx, lc->in.carve([&](Carve& k) { il.layout(k, lc->in_full, lc->in_scan); }));   // (reserved: no reallocation)
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
  ll_pose p; for (int k = 0; k < 4; k++) p.q_wxyz[k] = q_w_curr[k]; for (int k = 0; k < 3; k++) p.t[k] = t_w_curr[k];
  lc->poses.push_back(p);
  const int id = (int)lc->kfs.size() - 1;
  if (id >= 1) { ll_pg_edge e; pg_odometry_edge(&lc->poses[id - 1], id - 1, &lc->poses[id], id, &e); lc->edges.push_back(e); }
  ll_keyframe_info info;
  LL_TRY(ll_keyframe_analyze(ctx, lc->full, closing, c.incremental_cov, &info));
  std::vector<int> cand(id + 1);
  int nc = 0;
  LL_TRY(ll_loop_search(ctx, lc->kfs.data(), id + 1, id, &c.loop, nullptr, nullptr, cand.data(), &nc));
  cand.resize(nc);
  ll_loop_event* ke = log_push(lc, LL_LOOP_KEYFRAME);
  ke->ending_frame_idx = frame_index; ke->n_candidates = nc; ke->info = info;
  memcpy(ke->q_wxyz, p.q_wxyz, sizeof(p.q_wxyz)); memcpy(ke->t, p.t, sizeof(p.t));
  return loop_align(ctx, lc, cand);
}

}  // namespace

// Loop closure never fails the step: an error of its work other than LL_ERR_CUDA is logged (LL_LOOP_ERROR) and stops it for good.
int loop_step(ll_ctx* ctx, LoopClosure* lc, const double* d_pose, bool pushed, int frame_index, const double q_w_curr[4], const double t_w_curr[3]) {
  if (lc->closed || lc->stopped) return LL_OK;
  const int st = loop_step_work(ctx, lc, d_pose, pushed, frame_index, q_w_curr, t_w_curr);
  if (st == LL_OK || st == LL_ERR_CUDA) return st;
  ll_loop_event* e = log_push(lc, LL_LOOP_ERROR);
  e->status = st; e->ending_frame_idx = frame_index;
  lc->stopped = true;   // (the context's last error names the failure)
  return LL_OK;
}

int loop_read(LoopClosure* lc, ll_loop_event* out, int cap, int* n, int* n_dropped) {
  *n = 0;
  if (n_dropped) *n_dropped = 0;
  if (!lc) return LL_OK;
  const int k = (int)std::min((size_t)cap, lc->count);
  for (int i = 0; i < k; i++) out[i] = lc->ring[(lc->first + i) % lc->ring.size()];
  if (k > 0) { lc->first = (lc->first + k) % lc->ring.size(); lc->count -= k; }
  *n = k;
  if (n_dropped) *n_dropped = lc->dropped;
  lc->dropped = 0;
  return LL_OK;
}

int loop_result(const LoopClosure* lc, int* n, int* closed, ll_pose* poses_ori, ll_pose* poses_opt, int cap, ll_pg_edge* edge) {
  const int N = lc ? (int)lc->poses.size() : 0;
  if ((poses_ori || poses_opt) && cap < N) return LL_ERR_CAPACITY;
  if (n) *n = N;
  if (closed) *closed = lc && lc->closed ? 1 : 0;
  if (poses_ori && N) memcpy(poses_ori, lc->poses.data(), N * sizeof(ll_pose));
  if (poses_opt && N) memcpy(poses_opt, lc->closed ? lc->opt.data() : lc->poses.data(), N * sizeof(ll_pose));
  if (edge) { if (lc && lc->closed) *edge = lc->loop_edge; else memset(edge, 0, sizeof(*edge)); }
  return LL_OK;
}

int loop_cloud(ll_ctx* ctx, const LoopClosure* lc, int k, ll_point* out_host, size_t cap, size_t* n_out, const ll_point** out_dev) {
  if (!lc || !lc->closed) { ctx->set_error("no loop closed"); return LL_ERR_INVALID; }
  const int N = (int)lc->kfs.size();
  if (k < 0 || k >= N || (N - 1 - k) % 2 != 0) { ctx->set_error("keyframe k is not one the loop publishes (n - 1, n - 3, ...)"); return LL_ERR_INVALID; }
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
