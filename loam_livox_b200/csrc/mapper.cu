// Streaming odometry driver: Laser_mapping::process_new_scan + update_buff_for_matching (matching_mode 0 = sliding window of the last
// maximum_histroy_buffer feature clouds, the mode both shipped YAMLs select; matching_mode 1 = cells in range and in the FOV), with everything
// resident on the device (the history window, the cell maps, the match-map snapshot and its index, the features).
//
// Restates, on the reference side (ROS I/O, threads, mutexes and loop closure left out):
//   Laser_mapping::process_new_scan                loam_livox/source/laser_mapping.hpp:1316-1521
//   history window push / pop                      loam_livox/source/laser_mapping.hpp:1439-1487 (mode 0 concatenation :518-531)
//   Laser_mapping::update_buff_for_matching        loam_livox/source/laser_mapping.hpp:460-566 (mode 1 branch :471-516, whole-map VoxelGrid :533-537,
//                                                                                                  KdTreeFLANN build :544-545)
//   Laser_mapping::init_pointcloud_registration    loam_livox/source/laser_mapping.hpp:1266-1297
// The reference refreshes the match map on a background thread after every registered scan, with the pose of that scan; here the refresh
// runs at the start of the next scan (same pose, same map content), so the result is the reference's with maximum_parallel_thread = 1.
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "common.cuh"
#include "kernels.cuh"

static inline double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// m_laser_cloud_{corner,surface}_history (std::list<PointCloud>, :1446-1478) as ONE flat device array: the clouds of the window lie one after the
// other in push order, so the concatenation of mode 0 (:518-531) is the live range itself.  Two arenas, ping-pong: when the tail reaches the end of
// one, the live range is copied to the start of the other (no allocation per scan in steady state).
struct HistoryWindow {
  DevBuf buf[2]; int cur = 0;
  std::vector<std::pair<size_t, size_t>> segs;   // (offset, count) in points, oldest first
  size_t tail = 0;                               // first free point of buf[cur]
  size_t head() const { return segs.empty() ? tail : segs.front().first; }
  size_t live() const { return tail - head(); }
  const float4* data() const { return (const float4*)buf[cur].p + head(); }
  int push(ll_ctx* ctx, const float4* d_pts, size_t n) {
    cudaStream_t s = ctx->stream;
    const size_t cap = buf[cur].cap / 16;
    if (tail + n > cap) {   // slide: live range + the new cloud into the other arena
      const size_t need = live() + n;
      DevBuf& o = buf[cur ^ 1];
      LL_CUDA(ctx, cudaStreamSynchronize(s));   // (the other arena may be reallocated; nothing may still read it)
      LL_CUDA(ctx, o.reserve((need + need / 2 + 1024) * 16));
      const size_t h = head(), lv = live();
      if (lv) LL_CUDA(ctx, cudaMemcpyAsync(o.p, (const float4*)buf[cur].p + h, lv * 16, cudaMemcpyDeviceToDevice, s));
      for (auto& sg : segs) sg.first -= h;
      cur ^= 1; tail = lv;
    }
    if (n) LL_CUDA(ctx, cudaMemcpyAsync((float4*)buf[cur].p + tail, d_pts, n * 16, cudaMemcpyDeviceToDevice, s));
    segs.emplace_back(tail, n); tail += n;
    return LL_OK;
  }
  int reserve(ll_ctx* ctx, size_t points) { for (auto& b : buf) LL_CUDA(ctx, b.reserve_floor((points + points / 2 + 1024) * 16)); return LL_OK; }
  void pop_front() { if (!segs.empty()) segs.erase(segs.begin()); }
  void release() { buf[0].release(); buf[1].release(); segs.clear(); tail = 0; }
};

struct ll_mapper {
  ll_ctx* ctx = nullptr;
  HistoryWindow his_corner, his_surf;
  double last_his_add_q[4] = {1, 0, 0, 0}, last_his_add_t[3] = {0, 0, 0};   // m_last_his_add_q / _t (uninitialised members in the reference: defined as identity / 0)
  ll_mapper_config cfg;
  ll_cellmap* cells_corner = nullptr; ll_cellmap* cells_surf = nullptr;
  ll_map* match_map = nullptr;
  int frame_index = 0;
  double last_time_stamp = 0;   // m_last_time_stamp (laser_mapping.hpp:140)
  double q_w_curr[4] = {1, 0, 0, 0}, t_w_curr[3] = {0, 0, 0};
  DevBuf work;   // transformed / down-sampled feature clouds (work_layout)
  DevBuf snap;   // match-map snapshot clouds (corner, surf) between refreshes (snap_layout)
  int snap_n[2] = {0, 0}, fov[2] = {0, 0};
  bool have_map = false;
  bool map_dirty = false;   // m_if_mapping_updated_{corner,surface}
  bool trace = false;       // LL_MAPPER_TRACE=1
  // the piecewise front end (FrameLayout; segmented VoxelGrid scratch of its main / corner chain).  Two arenas: ll_mapper_process_frames reads
  // frame f's pieces out of frame[f & 1] while the front end of frame f + 1 fills the other; ll_mapper_process_frame uses frame[0].
  DevBuf frame[2], frame_vg[2];
  FrontGraph frame_graph[2];   // the device part of the front end, replayed per arena
  int frame_pieces = 0;        // the pieces `frame` was laid out for
};

// frame: the front end's device record and, per class, the gathered piece segments and the first VoxelGrid's outputs
struct FrameLayout {
  FrameDev* dev; float4* cls[2]; float4* mid[2];
  void layout(Carve& k, size_t cap) { dev = k.take<FrameDev>(1); for (int c = 0; c < 2; c++) { cls[c] = k.take<float4>(cap); mid[c] = k.take<float4>(cap); } }
};

// snap: the match-map snapshot (the two whole-map VoxelGrid outputs) and their counts
struct SnapLayout {
  float4* c; float4* s; int* cnt;
  void layout(Carve& k, size_t mc, size_t ms) { c = k.take<float4>(mc + 1); s = k.take<float4>(ms + 1); cnt = k.take<int>(2); }
};
// work: a scan's features in the world frame (w2 corner, w3 surface), down-sampled (w0, w1), their counts and the pose
struct WorkLayout {
  float4* w0; float4* w1; float4* w2; float4* w3; int* cnt; double* pose;
  void layout(Carve& k, size_t n) { w0 = k.take<float4>(n); w1 = k.take<float4>(n); w2 = k.take<float4>(n); w3 = k.take<float4>(n); cnt = k.take<int>(2); pose = k.take<double>(7); }
};

// Every buffer whose size follows the map is allocated here, once, for the configured reservation (a reallocation inside a scan call
// synchronises the device and stalls that call for far longer than the scan takes; one such stall per doubling of the map dominates the mean
// scan time of a long stream).  Past the reservation everything still grows by doubling.
static int mapper_reserve(ll_ctx* ctx, ll_mapper* m) {
  const size_t R = (size_t)(m->cfg.reserve_map_points > 0 ? m->cfg.reserve_map_points : 0), S = (size_t)(m->cfg.reserve_store_points > 0 ? m->cfg.reserve_store_points : 0);
  const int F = ctx->cfg.max_features;
  WorkLayout w; LL_CUDA(ctx, m->work.reserve_floor(layout_bytes([&](Carve& c) { w.layout(c, F); })));
  // the piecewise front end: pieces x max_scan_points per class (overlapping pieces repeat points), nothing allocated per frame
  { const int P = m->cfg.pipeline.pieces >= 1 && m->cfg.pipeline.pieces <= LL_MAX_PIECES ? m->cfg.pipeline.pieces : 1;
    const size_t cap = (size_t)P * ctx->cfg.max_scan_points;
    FrameLayout fl; for (DevBuf& b : m->frame) LL_CUDA(ctx, b.reserve_floor(layout_bytes([&](Carve& c) { fl.layout(c, cap); })));
    for (DevBuf& b : m->frame_vg) LL_CUDA(ctx, b.reserve_floor(std::max(voxel_grid_bytes((int)cap, P), voxel_grid_bytes(ctx->cfg.max_scan_points, 1))));
    m->frame_pieces = P; }
  if (S) { LL_TRY(ll_cellmap_reserve(ctx, m->cells_corner, S, F)); LL_TRY(ll_cellmap_reserve(ctx, m->cells_surf, S, F)); }
  // The two map-side arenas, each at the largest of its consumers.  Both: the append's VoxelGrid of a scan's features (corner half on stream2 /
  // scratch2, surface half on the context's stream / scratch) and the refresh's whole-map VoxelGrid and index build (the halves side by side
  // the same way).  scratch alone: the registration's query sort and K10 hash set.
  size_t side = voxel_grid_bytes(F);
  if (R) side = std::max(side, std::max(voxel_grid_bytes((int)R), tree_scratch_bytes((int)R)));
  const size_t reg = std::max(query_sort_bytes(F, 1), layout_bytes([&](Carve& c) { l1_set_layout(c, F); }));
  LL_CUDA(ctx, ctx->scratch.reserve_floor(std::max(side, reg)));
  LL_CUDA(ctx, ctx->scratch2.reserve_floor(side));
  if (!R) return LL_OK;
  LL_TRY(m->his_corner.reserve(ctx, R)); LL_TRY(m->his_surf.reserve(ctx, R));
  SnapLayout sn; LL_CUDA(ctx, m->snap.reserve_floor(layout_bytes([&](Carve& c) { sn.layout(c, R, R); })));
  for (BucketTree* t : {&m->match_map->corner, &m->match_map->surf}) LL_CUDA(ctx, t->storage.reserve_floor(tree_storage_bytes((int)R)));
  return LL_OK;
}

extern "C" {

void ll_mapper_release(ll_mapper* m);

void ll_mapper_config_default(ll_mapper_config* c) {
  memset(c, 0, sizeof(*c));
  c->line_resolution = 0.1f; c->plane_resolution = 0.4f;             // performance_precision.yaml:12-13
  c->cell_resolution = 1.0f; c->threshold_cell_revisit = 2000;      // laser_mapping.hpp:272, performance_precision.yaml
  c->maximum_search_range_corner = 100.f; c->maximum_search_range_surface = 100.f; c->maximum_in_fov_angle = 45.f;   // :691-695
  c->down_sample_replace = 1;                                        // :277
  c->matching_mode = 0; c->maximum_history_size = 400;               // mapping/matching_mode, mapping/maximum_histroy_buffer (performance_precision.yaml:28-29)
  c->pipeline.pieces = 3; c->pipeline.use_piece = 0; c->pipeline.whole_frame = 1;
  c->pipeline.extractor_leaf_corner = 0.1f; c->pipeline.extractor_leaf_surf = 0.2f; c->pipeline.mapping_leaf_corner = 0.1f; c->pipeline.mapping_leaf_surf = 0.4f;
  ll_reg_state_default(&c->reg);
  c->max_cells = 0;
  c->reserve_map_points = 1 << 22; c->reserve_store_points = 1 << 22;   // window of 400 clouds x up to ~10k down-sampled features; see mapper_reserve
}

int ll_mapper_create(ll_ctx* ctx, const ll_mapper_config* cfg, ll_mapper** out) {
  if (!ctx || !cfg || !out) return LL_ERR_INVALID;
  ll_mapper* m = new ll_mapper(); m->ctx = ctx; m->cfg = *cfg;
  int st = ll_cellmap_create(ctx, cfg->cell_resolution, cfg->threshold_cell_revisit, cfg->max_cells, &m->cells_corner);
  if (st == LL_OK) st = ll_cellmap_create(ctx, cfg->cell_resolution, cfg->threshold_cell_revisit, cfg->max_cells, &m->cells_surf);
  if (st != LL_OK) { ll_cellmap_release(m->cells_corner); delete m; return st; }
  for (int k = 0; k < 4; k++) m->q_w_curr[k] = cfg->reg.q_w_curr[k];
  for (int k = 0; k < 3; k++) m->t_w_curr[k] = cfg->reg.t_w_curr[k];
  ll_extract_reset(ctx);
  { const char* e = getenv("LL_MAPPER_TRACE"); m->trace = e && e[0] == '1'; }
  m->match_map = new ll_map(); m->match_map->device = ctx->device;   // indexed in place by every refresh (ll_map_rebuild)
  st = mapper_reserve(ctx, m);
  if (st == LL_OK && ll_ctx_warmup(ctx) == LL_ERR_CUDA) st = LL_ERR_CUDA;   // the first registered scan of a stream is not the one that loads the kernels
  if (st != LL_OK) { ll_mapper_release(m); return st; }
  *out = m; return LL_OK;
}
void ll_mapper_release(ll_mapper* m) {
  if (!m) return;
  cudaSetDevice(m->ctx->device);
  ll_cellmap_release(m->cells_corner); ll_cellmap_release(m->cells_surf);
  if (m->match_map) ll_map_release(m->match_map);
  m->work.release(); m->snap.release(); m->his_corner.release(); m->his_surf.release();
  for (FrontGraph& g : m->frame_graph) if (g.exec) cudaGraphExecDestroy(g.exec);
  m->frame[0].release(); m->frame[1].release(); m->frame_vg[0].release(); m->frame_vg[1].release(); delete m;
}
int ll_mapper_pose(const ll_mapper* m, double q_wxyz[4], double t[3], int* frame_index) {
  if (!m) return LL_ERR_INVALID;
  for (int k = 0; k < 4; k++) q_wxyz[k] = m->q_w_curr[k]; for (int k = 0; k < 3; k++) t[k] = m->t_w_curr[k];
  if (frame_index) *frame_index = m->frame_index;
  return LL_OK;
}

static void out_init(const ll_mapper* m, ll_reg_result* out) {
  memset(out, 0, sizeof(*out)); out->status = 1;
  for (int k = 0; k < 4; k++) out->q_w_curr[k] = m->q_w_curr[k]; for (int k = 0; k < 3; k++) out->t_w_curr[k] = m->t_w_curr[k];
}

// One mapper step on features already in A.feat (nc corners, then ns surfaces) whose full cloud's largest time stamp is max_t: (refresh the
// match map) -> registration -> world-frame features -> VoxelGrid -> history window and cell maps -> pose.  Every registered scan of
// ll_mapper_process_scan and every published piece of ll_mapper_process_frame goes through it.
static int mapper_step(ll_mapper* m, int nc, int ns, double max_t, ll_reg_result* out, ll_mapper_stats* stats) {
  ll_ctx* ctx = m->ctx;
  cudaStream_t s = ctx->stream;
  const RegArrays& A = ctx->A;
  out_init(m, out);
  double tp = now_ms();
  // :1336-1350: the time-stamp range of this scan comes from the full cloud (min of refine_blur = the previous scan's maximum), and
  // init_pointcloud_registration copies m_current_frame_index BEFORE it is incremented
  const int frame_index_for_reg = m->frame_index;
  const double minimum_pt_time_stamp = m->last_time_stamp, maximum_pt_time_stamp = max_t;
  m->last_time_stamp = maximum_pt_time_stamp;
  m->frame_index++;                                                              // m_current_frame_index++ (:1350)
  // ---- update_buff_for_matching (mode 1): snapshot of the cells in range and in the FOV, whole-map VoxelGrid, index
  if (m->map_dirty) {
    size_t mc = 0, ms = 0; const ll_point* d_mc = nullptr; const ll_point* d_ms = nullptr; int fov_c = 0, fov_s = 0;
    if (m->cfg.matching_mode == 0) {   // :518-531: the concatenation of the history window (the live range of the flat array)
      mc = m->his_corner.live(); ms = m->his_surf.live(); d_mc = (const ll_point*)m->his_corner.data(); d_ms = (const ll_point*)m->his_surf.data();
    } else {
    LL_TRY(ll_cellmap_assemble(ctx, m->cells_corner, m->q_w_curr, m->t_w_curr, m->cfg.maximum_search_range_corner, m->cfg.maximum_in_fov_angle, m->cfg.line_resolution,
                               m->cfg.down_sample_replace, nullptr, 0, &mc, &fov_c, &d_mc));
    LL_TRY(ll_cellmap_assemble(ctx, m->cells_surf, m->q_w_curr, m->t_w_curr, m->cfg.maximum_search_range_surface, m->cfg.maximum_in_fov_angle, m->cfg.plane_resolution,
                               m->cfg.down_sample_replace, nullptr, 0, &ms, &fov_s, &d_ms));
    }
    SnapLayout sn; LL_CUDA(ctx, m->snap.carve([&](Carve& c) { sn.layout(c, mc, ms); }));
    float4* s0 = sn.c; float4* s1 = sn.s; int* d_sc = sn.cnt;
    int hc[2] = {0, 0};
    // the two whole-map VoxelGrids side by side (corner on the side stream with its own scratch)
    cudaStream_t s2 = ctx->stream2;
    LL_CUDA(ctx, cudaEventRecord(ctx->sev.fork, s)); LL_CUDA(ctx, cudaStreamWaitEvent(s2, ctx->sev.fork, 0));
    if (mc > 0) LL_TRY(launch_voxel_grid(ctx, s2, ctx->scratch2, (const float4*)d_mc, (int)mc, nullptr, m->cfg.line_resolution, s0, d_sc)); else LL_CUDA(ctx, cudaMemsetAsync(d_sc, 0, 4, s2));      // :533-534
    if (ms > 0) LL_TRY(launch_voxel_grid(ctx, s, ctx->scratch, (const float4*)d_ms, (int)ms, nullptr, m->cfg.plane_resolution, s1, d_sc + 1)); else LL_CUDA(ctx, cudaMemsetAsync(d_sc + 1, 0, 4, s));   // :536-537
    LL_CUDA(ctx, cudaEventRecord(ctx->sev.join, s2)); LL_CUDA(ctx, cudaStreamWaitEvent(s, ctx->sev.join, 0));
    LL_CUDA(ctx, cudaMemcpyAsync(hc, d_sc, 8, cudaMemcpyDeviceToHost, s));
    LL_CUDA(ctx, cudaStreamSynchronize(s));
    m->have_map = false;
    if (hc[0] > 0 && hc[1] > 0) {
      LL_TRY(ll_map_rebuild(ctx, m->match_map, s0, (size_t)hc[0], s1, (size_t)hc[1], LL_FMT_XYZI16, LL_DEVICE));   // buffers reused: no allocation per scan
      m->have_map = true;
    }                      // :544-545
    m->snap_n[0] = hc[0]; m->snap_n[1] = hc[1]; m->fov[0] = fov_c; m->fov[1] = fov_s;
    m->map_dirty = false;
  }
  if (stats) { stats->ms_refresh = (float)(now_ms() - tp); stats->map_corner = m->snap_n[0]; stats->map_surf = m->snap_n[1]; stats->cells_in_fov_corner = m->fov[0]; stats->cells_in_fov_surf = m->fov[1]; }
  WorkLayout wl; LL_CUDA(ctx, m->work.carve([&](Carve& c) { wl.layout(c, (size_t)(nc > ns ? nc : ns)); }));
  float4* w0 = wl.w0; float4* w1 = wl.w1; float4* w2 = wl.w2; float4* w3 = wl.w3; int* d_cnt = wl.cnt;
  int hc[2] = {0, 0};
  // ---- init_pointcloud_registration + find_out_incremental_transfrom (:1266-1297, :1405)
  ll_reg_state st = m->cfg.reg;
  st.current_frame_index = frame_index_for_reg;
  st.minimum_pt_time_stamp = minimum_pt_time_stamp; st.maximum_pt_time_stamp = maximum_pt_time_stamp;   // :1287-1288
  st.rng_seed = m->cfg.reg.rng_seed + frame_index_for_reg;   // a fresh Point_cloud_registration (and m_rand_float) per scan (:1348)
  for (int k = 0; k < 4; k++) { st.q_w_last[k] = m->q_w_curr[k]; st.q_w_curr[k] = m->q_w_curr[k]; }
  for (int k = 0; k < 3; k++) { st.t_w_last[k] = m->t_w_curr[k]; st.t_w_curr[k] = m->t_w_curr[k]; }
  st.para_buffer_incremental[0] = st.para_buffer_incremental[1] = st.para_buffer_incremental[2] = 0; st.para_buffer_incremental[3] = 1;
  st.para_buffer_incremental[4] = st.para_buffer_incremental[5] = st.para_buffer_incremental[6] = 0;
  tp = now_ms();
  if (m->have_map) LL_TRY(register_device(ctx, m->match_map, nc, ns, &st, out));
  if (stats) stats->ms_register = (float)(now_ms() - tp);
  tp = now_ms();   // no map yet: the gate of :199 returns 1
  if (out->status == 0) return LL_OK;                                           // rejected: frame discarded (:1413-1416)
  // ---- new features to the world frame (:1422-1432), VoxelGrid (:1434-1437), cell maps (:1492-1493)
  double* h = ctx->pin->mapper_pose; for (int k = 0; k < 4; k++) h[k] = out->q_w_curr[k]; for (int k = 0; k < 3; k++) h[4 + k] = out->t_w_curr[k];
  double* d_pose = wl.pose;
  LL_CUDA(ctx, cudaMemcpyAsync(d_pose, h, 7 * sizeof(double), cudaMemcpyHostToDevice, s));
  {
    cudaStream_t s2 = ctx->stream2;
    LL_CUDA(ctx, cudaEventRecord(ctx->sev.fork, s)); LL_CUDA(ctx, cudaStreamWaitEvent(s2, ctx->sev.fork, 0));
    if (nc > 0) { LL_TRY(launch_transform(ctx, s2, d_pose, A.feat, nc, w2)); LL_TRY(launch_voxel_grid(ctx, s2, ctx->scratch2, w2, nc, nullptr, m->cfg.line_resolution, w0, d_cnt)); } else LL_CUDA(ctx, cudaMemsetAsync(d_cnt, 0, 4, s2));
    if (ns > 0) { LL_TRY(launch_transform(ctx, s, d_pose, A.feat + nc, ns, w3)); LL_TRY(launch_voxel_grid(ctx, s, ctx->scratch, w3, ns, nullptr, m->cfg.plane_resolution, w1, d_cnt + 1)); } else LL_CUDA(ctx, cudaMemsetAsync(d_cnt + 1, 0, 4, s));
    LL_CUDA(ctx, cudaEventRecord(ctx->sev.join, s2)); LL_CUDA(ctx, cudaStreamWaitEvent(s, ctx->sev.join, 0));
  }
  LL_CUDA(ctx, cudaMemcpyAsync(hc, d_cnt, 8, cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  const double tr0 = now_ms();
  // history window (:1439-1478): r_diff / t_diff compare the pose adopted from the PREVIOUS scan (m_q_w_curr is only overwritten at :1498) with the
  // pose of the last addition; history_add_t_step = history_add_angle_step = 0 (:83-84)
  {
    const double* q = m->q_w_curr; const double* lq = m->last_his_add_q;
    double dot = fabs(q[0] * lq[0] + q[1] * lq[1] + q[2] * lq[2] + q[3] * lq[3]); if (dot > 1.0) dot = 1.0;
    const double r_diff = 2.0 * acos(dot) * 57.3;
    double t2 = 0; for (int k = 0; k < 3; k++) t2 += (m->t_w_curr[k] - m->last_his_add_t[k]) * (m->t_w_curr[k] - m->last_his_add_t[k]);
    const double t_diff = sqrt(t2);
    if ((int)m->his_corner.segs.size() < m->cfg.maximum_history_size || t_diff > 0.0 || r_diff > 0.0 * 57.3) {
      for (int k = 0; k < 4; k++) m->last_his_add_q[k] = m->q_w_curr[k]; for (int k = 0; k < 3; k++) m->last_his_add_t[k] = m->t_w_curr[k];
      LL_TRY(m->his_corner.push(ctx, w0, (size_t)hc[0]));
      LL_TRY(m->his_surf.push(ctx, w1, (size_t)hc[1]));
    }
    if ((int)m->his_corner.segs.size() > m->cfg.maximum_history_size) m->his_corner.pop_front();
    if ((int)m->his_surf.segs.size() > m->cfg.maximum_history_size) m->his_surf.pop_front();
  }
  const double tr1 = now_ms();
  LL_TRY(ll_cellmap_append(ctx, m->cells_corner, w0, (size_t)hc[0], LL_FMT_XYZI16, LL_DEVICE));
  const double tr2 = now_ms();
  LL_TRY(ll_cellmap_append(ctx, m->cells_surf, w1, (size_t)hc[1], LL_FMT_XYZI16, LL_DEVICE));
  if (m->trace && now_ms() - tp > 10.0)   // LL_MAPPER_TRACE=1: where a slow append went (transform + VoxelGrid + sync | history | corner cells | surface cells)
    fprintf(stderr, "ll_mapper trace: frame %d append %.2f ms = features %.2f + history %.2f + cells %.2f + %.2f\n", m->frame_index, now_ms() - tp, tr0 - tp, tr1 - tr0, tr2 - tr1, now_ms() - tr2);
  m->map_dirty = true;                                                           // m_if_mapping_updated_* (:1490-1491)
  if (stats) { stats->appended_corner = hc[0]; stats->appended_surf = hc[1]; stats->ms_append = (float)(now_ms() - tp); }
  for (int k = 0; k < 4; k++) m->q_w_curr[k] = out->q_w_curr[k]; for (int k = 0; k < 3; k++) m->t_w_curr[k] = out->t_w_curr[k];   // :1496-1505
  return LL_OK;
}

// One scan: features -> mapper_step.
int ll_mapper_process_scan(ll_mapper* m, const void* raw, size_t n, int fmt, int where, double stamp, ll_reg_result* out, ll_mapper_stats* stats) {
  if (!m || !out) return LL_ERR_INVALID;
  ll_ctx* ctx = m->ctx; cudaSetDevice(ctx->device);
  if (stats) memset(stats, 0, sizeof(*stats));
  const double tp = now_ms();
  int nc = 0, ns = 0, dropped = 0;
  LL_TRY(scan_front_end(ctx, raw, n, fmt, where, stamp, &m->cfg.pipeline, &nc, &ns, &dropped));
  out_init(m, out);
  if (stats) { stats->n_corner = nc; stats->n_surf = ns; stats->ms_front_end = (float)(now_ms() - tp); }
  if (dropped) return LL_OK;                                                     // laser_feature_extractor.hpp:287
  return mapper_step(m, nc, ns, (double)ctx->last_full_max_t, out, stats);
}

}  // extern "C"

// The pieces a frame is cut into and the entries it publishes; LL_ERR_INVALID for a bad odom_mode, pieces or cap.
static int frame_publish(ll_mapper* m, int odom_mode, int cap, int* pieces, int* publish) {
  ll_ctx* ctx = m->ctx;
  *pieces = m->cfg.reg.if_motion_deblur ? 1 : m->cfg.pipeline.pieces;   // laser_feature_extractor.hpp:305-309
  if (*pieces < 1 || *pieces > m->frame_pieces) { ctx->set_error("pieces must be 1 ... 16"); return LL_ERR_INVALID; }
  if (odom_mode != 0 && odom_mode != 1) { ctx->set_error("odom_mode must be 0 or 1"); return LL_ERR_INVALID; }
  *publish = odom_mode ? *pieces : 1;                                            // :385-388
  if (cap < *publish) { ctx->set_error("cap smaller than the pieces to publish"); return LL_ERR_INVALID; }
  return LL_OK;
}
static int frame_arena(ll_mapper* m, int a, FrameArena* fa) {
  ll_ctx* ctx = m->ctx;
  const int cap = m->frame_pieces * ctx->cfg.max_scan_points;
  FrameLayout fl; LL_CUDA(ctx, m->frame[a].carve([&](Carve& c) { fl.layout(c, (size_t)cap); }));
  *fa = FrameArena{fl.dev, {fl.cls[0], fl.cls[1]}, {fl.mid[0], fl.mid[1]}, cap, {&m->frame_vg[0], &m->frame_vg[1]}, &m->frame_graph[a]};
  return LL_OK;
}
// First published piece of a completed front end whose features exceed max_features (publish: none).
static int first_piece_over(const ll_mapper* m, const FrameOut& fo, int publish) {
  for (int i = 0; i < publish; i++) {
    const int nc = fo.out_end[0][i] - (i ? fo.out_end[0][i - 1] : 0), nsf = fo.out_end[1][i] - (i ? fo.out_end[1][i - 1] : 0);
    if (nc + nsf > m->ctx->cfg.max_features) return i;
  }
  return publish;
}

// The published pieces of a frame whose front end has completed (fo: its read-back; fa: its arena): per piece its features into A.feat and
// mapper_step.  A rejected piece leaves the pose as it was, and the next piece continues from there.  `copied` runs once piece 0's features
// are enqueued for copying; free_ev (may be null) is recorded behind the last copy out of `fa`.
template <typename F>
static int frame_pieces(ll_mapper* m, const FrameArena& fa, const FrameOut& fo, int publish, float ms_front_end, ll_reg_result* out, ll_mapper_stats* stats,
                        int* n_pieces, cudaEvent_t free_ev, F&& copied) {
  ll_ctx* ctx = m->ctx;
  for (int i = 0; i < publish; i++) {
    const int c0 = i ? fo.out_end[0][i - 1] : 0, s0 = i ? fo.out_end[1][i - 1] : 0;
    const int nc = fo.out_end[0][i] - c0, nsf = fo.out_end[1][i] - s0;
    ll_mapper_stats* st = stats ? stats + i : nullptr;
    if (st) { memset(st, 0, sizeof(*st)); st->n_corner = nc; st->n_surf = nsf; st->ms_front_end = i == 0 ? ms_front_end : 0.f; }
    out_init(m, out + i);
    if (nc + nsf > ctx->cfg.max_features) { ctx->set_error("more features than max_features"); return LL_ERR_CAPACITY; }
    LL_CUDA(ctx, cudaMemcpyAsync(ctx->A.feat, fa.cls[0] + c0, (size_t)nc * 16, cudaMemcpyDeviceToDevice, ctx->stream));
    LL_CUDA(ctx, cudaMemcpyAsync(ctx->A.feat + nc, fa.cls[1] + s0, (size_t)nsf * 16, cudaMemcpyDeviceToDevice, ctx->stream));
    if (free_ev && i == publish - 1) LL_CUDA(ctx, cudaEventRecord(free_ev, ctx->stream));
    if (i == 0) LL_TRY(copied());
    LL_TRY(mapper_step(m, nc, nsf, (double)ll_ord2f(fo.tmax[i]), out + i, st));
    *n_pieces = i + 1;
  }
  return LL_OK;
}

// One frame: the piecewise front end (every head, every piece, one host read), then per published piece its features into A.feat and
// mapper_step.
extern "C" int ll_mapper_process_frame(ll_mapper* m, int n_heads, const void* const* raws, const size_t* ns, int fmt, int where, const double* stamps,
                                       int odom_mode, ll_reg_result* out, ll_mapper_stats* stats, int cap, int* n_pieces) {
  if (!m || !out || !raws || !ns || !stamps || !n_pieces || n_heads < 1 || n_heads > LL_MAX_HEADS) return LL_ERR_INVALID;
  *n_pieces = 0;
  ll_ctx* ctx = m->ctx; cudaSetDevice(ctx->device);
  int pieces = 0, publish = 0;
  LL_TRY(frame_publish(m, odom_mode, cap, &pieces, &publish));
  size_t total = 0;
  for (int h = 0; h < n_heads; h++) { if (!raws[h] && ns[h]) return LL_ERR_INVALID; total += ns[h]; }
  if (total > (size_t)ctx->cfg.max_scan_points) { ctx->set_error("frame (all heads) larger than max_scan_points"); return LL_ERR_CAPACITY; }
  const double tp = now_ms();
  FrameArena fa; LL_TRY(frame_arena(m, 0, &fa));
  LL_TRY(frame_front_end(ctx, ctx->own_front(), fa, n_heads, raws, ns, fmt, where, stamps, pieces, &m->cfg.pipeline));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const FrameOut fo = ctx->pin->frame;
  const float ms_front_end = (float)(now_ms() - tp);
  if (fo.heads_live == 0) return LL_OK;                                          // laser_feature_extractor.hpp:287, every head
  return frame_pieces(m, fa, fo, publish, ms_front_end, out, stats, n_pieces, nullptr, [] { return LL_OK; });
}

// ---------------------------------------------------------------------------------------------- sequences
// The front end of input k + 1 is enqueued on the context's front-end streams (ll_ctx::fe_stream) before the mapper step(s) of input k, so it
// runs under them.  Nothing the mapper step reads or writes is touched by the front end, whose results only reach the mapper through the copy
// into A.feat; the extractor's host bookkeeping advances in input order.  So every result is the one-by-one calls'.
//
// A front end enqueued ahead of an input that then fails: it is drained (it reads the caller's inputs) and its host bookkeeping undone, so that
// the extractor stands where the one-by-one calls leave it.
struct Ahead { ExtractState saved; bool on = false; };
static void sequence_unwind(ll_ctx* ctx, const Ahead& a) {
  const FrontStreams fs = ctx->pipe_front();
  for (cudaStream_t s : {fs.main, fs.corner, fs.petals}) cudaStreamSynchronize(s);
  if (a.on) ctx->ex = a.saved;
}
static int check_format(ll_ctx* ctx, int fmt, int where) {
  if ((fmt != LL_FMT_XYZI16 && fmt != LL_FMT_PCL32 && fmt != LL_FMT_STRIDED) || (where != LL_HOST && where != LL_DEVICE)) {
    ctx->set_error("unknown point format or memory kind"); return LL_ERR_INVALID;
  }
  return LL_OK;
}
// Host records are staged in stage_in: reserved for max_scan_points records before the first front end, because a reallocation (cudaFree)
// would synchronise the device in the middle of the sequence.
static int reserve_stage(ll_ctx* ctx, int fmt, int where) {
  if (where != LL_HOST || fmt == LL_FMT_XYZI16) return LL_OK;
  const size_t rec = fmt == LL_FMT_PCL32 ? 32 : (size_t)ctx->layout.point_step;
  LL_CUDA(ctx, ctx->stage_in.reserve((size_t)ctx->cfg.max_scan_points * rec));
  return LL_OK;
}

static int frames_run(ll_mapper* m, int n_frames, int n_heads, const void* const* raws, const size_t* ns, int fmt, int where, const double* stamps,
                      int pieces, int publish, ll_reg_result* out, ll_mapper_stats* stats, int cap, int* n_pieces, int* done, Ahead& ahead) {
  ll_ctx* ctx = m->ctx;
  const FrontStreams fs = ctx->pipe_front();
  FrameArena fa[2]; LL_TRY(frame_arena(m, 0, &fa[0])); LL_TRY(frame_arena(m, 1, &fa[1]));
  auto enqueue = [&](int f) -> int {   // frame f's front end into arena f & 1, behind the last copy out of it (frame f - 2's)
    const size_t o = (size_t)f * n_heads;
    LL_CUDA(ctx, cudaStreamWaitEvent(fs.main, ctx->sev.fe_free[f & 1], 0));
    LL_TRY(frame_front_end(ctx, fs, fa[f & 1], n_heads, raws + o, ns + o, fmt, where, stamps + o, pieces, &m->cfg.pipeline));
    LL_CUDA(ctx, cudaEventRecord(ctx->sev.fe_ready, fs.main));
    return LL_OK;
  };
  double t = now_ms();
  LL_TRY(enqueue(0));
  float ms_enqueue = (float)(now_ms() - t);
  for (int f = 0; f < n_frames; f++) {
    ahead.on = false;
    t = now_ms();
    LL_CUDA(ctx, cudaEventSynchronize(ctx->sev.fe_ready));
    const FrameOut fo = ctx->pin->frame;   // read before the next front end is enqueued (PinnedStage)
    const float ms_front_end = ms_enqueue + (float)(now_ms() - t);
    // the next front end goes under this frame's steps unless one of its pieces will stop the sequence
    const bool next = f + 1 < n_frames && (fo.heads_live == 0 || first_piece_over(m, fo, publish) == publish);
    auto enqueue_next = [&]() -> int {
      if (!next) return LL_OK;
      ahead.saved = ctx->ex; ahead.on = true;
      const double t1 = now_ms();
      LL_TRY(enqueue(f + 1));
      ms_enqueue = (float)(now_ms() - t1);
      return LL_OK;
    };
    if (fo.heads_live == 0) LL_TRY(enqueue_next());                             // laser_feature_extractor.hpp:287, every head
    else LL_TRY(frame_pieces(m, fa[f & 1], fo, publish, ms_front_end, out + (size_t)f * cap, stats ? stats + (size_t)f * cap : nullptr, &n_pieces[f],
                             ctx->sev.fe_free[f & 1], enqueue_next));
    *done = f + 1;
  }
  return LL_OK;
}

extern "C" int ll_mapper_process_frames(ll_mapper* m, int n_frames, int n_heads, const void* const* raws, const size_t* ns, int fmt, int where,
                                        const double* stamps, int odom_mode, ll_reg_result* out, ll_mapper_stats* stats, int cap, int* n_pieces, int* n_frames_done) {
  if (n_frames_done) *n_frames_done = 0;
  if (!m || !out || !raws || !ns || !stamps || !n_pieces || !n_frames_done || n_frames < 1 || n_heads < 1 || n_heads > LL_MAX_HEADS) return LL_ERR_INVALID;
  ll_ctx* ctx = m->ctx; cudaSetDevice(ctx->device);
  int pieces = 0, publish = 0;
  LL_TRY(frame_publish(m, odom_mode, cap, &pieces, &publish));
  LL_TRY(check_format(ctx, fmt, where));
  const size_t n_in = (size_t)n_frames * n_heads;
  for (size_t k = 0; k < n_in; k++) if (!raws[k] && ns[k]) { ctx->set_error("null cloud of " + std::to_string(ns[k]) + " points"); return LL_ERR_INVALID; }
  for (int f = 0; f < n_frames; f++) {
    size_t total = 0; for (int h = 0; h < n_heads; h++) total += ns[(size_t)f * n_heads + h];
    if (total > (size_t)ctx->cfg.max_scan_points) { ctx->set_error("frame " + std::to_string(f) + " (all heads) larger than max_scan_points"); return LL_ERR_CAPACITY; }
  }
  LL_TRY(reserve_stage(ctx, fmt, where));
  for (int f = 0; f < n_frames; f++) n_pieces[f] = 0;
  Ahead ahead; int done = 0;
  const int st = frames_run(m, n_frames, n_heads, raws, ns, fmt, where, stamps, pieces, publish, out, stats, cap, n_pieces, &done, ahead);
  if (st != LL_OK) sequence_unwind(ctx, ahead);
  *n_frames_done = done;
  return st;
}

static int scans_run(ll_mapper* m, int n_scans, const void* const* raws, const size_t* ns, int fmt, int where, const double* stamps, ll_reg_result* out,
                     ll_mapper_stats* stats, int* done, Ahead& ahead) {
  ll_ctx* ctx = m->ctx;
  const FrontStreams fs = ctx->pipe_front();
  const ll_pipeline_cfg* pc = &m->cfg.pipeline;
  auto enqueue = [&](int k) -> int {   // behind the copy of scan k - 1's features out of tmp_a / tmp_b
    LL_CUDA(ctx, cudaStreamWaitEvent(fs.main, ctx->sev.fe_free[0], 0));
    LL_TRY(scan_front_end_enqueue(ctx, fs, raws[k], ns[k], fmt, where, stamps[k], pc));
    LL_CUDA(ctx, cudaEventRecord(ctx->sev.fe_ready, fs.main));
    return LL_OK;
  };
  double t = now_ms();
  LL_TRY(enqueue(0));
  float ms_enqueue = (float)(now_ms() - t);
  for (int k = 0; k < n_scans; k++) {
    ahead.on = false;
    ll_mapper_stats* st = stats ? stats + k : nullptr;
    if (st) memset(st, 0, sizeof(*st));
    t = now_ms();
    LL_CUDA(ctx, cudaEventSynchronize(ctx->sev.fe_ready));
    int nc = 0, nsf = 0, dropped = 0;
    LL_TRY(scan_front_end_finish(ctx, ctx->stream, pc, &nc, &nsf, &dropped));   // reads the pinned counts before the next front end is enqueued
    LL_CUDA(ctx, cudaEventRecord(ctx->sev.fe_free[0], ctx->stream));
    const float ms_front_end = ms_enqueue + (float)(now_ms() - t);
    if (k + 1 < n_scans) {
      ahead.saved = ctx->ex; ahead.on = true;
      const double t1 = now_ms();
      LL_TRY(enqueue(k + 1));
      ms_enqueue = (float)(now_ms() - t1);
    }
    out_init(m, out + k);
    if (st) { st->n_corner = nc; st->n_surf = nsf; st->ms_front_end = ms_front_end; }
    if (!dropped) LL_TRY(mapper_step(m, nc, nsf, (double)ctx->last_full_max_t, out + k, st));   // laser_feature_extractor.hpp:287
    *done = k + 1;
  }
  return LL_OK;
}

extern "C" int ll_mapper_process_scans(ll_mapper* m, int n_scans, const void* const* raws, const size_t* ns, int fmt, int where, const double* stamps,
                                       ll_reg_result* out, ll_mapper_stats* stats, int* n_scans_done) {
  if (n_scans_done) *n_scans_done = 0;
  if (!m || !out || !raws || !ns || !stamps || !n_scans_done || n_scans < 1) return LL_ERR_INVALID;
  ll_ctx* ctx = m->ctx; cudaSetDevice(ctx->device);
  LL_TRY(check_format(ctx, fmt, where));
  for (int k = 0; k < n_scans; k++) if (!raws[k] && ns[k]) { ctx->set_error("null cloud of " + std::to_string(ns[k]) + " points"); return LL_ERR_INVALID; }
  for (int k = 0; k < n_scans; k++) if (ns[k] > (size_t)ctx->cfg.max_scan_points) { ctx->set_error("scan " + std::to_string(k) + " larger than max_scan_points"); return LL_ERR_CAPACITY; }
  LL_TRY(reserve_stage(ctx, fmt, where));
  Ahead ahead; int done = 0;
  const int st = scans_run(m, n_scans, raws, ns, fmt, where, stamps, out, stats, &done, ahead);
  if (st != LL_OK) sequence_unwind(ctx, ahead);
  *n_scans_done = done;
  return st;
}
