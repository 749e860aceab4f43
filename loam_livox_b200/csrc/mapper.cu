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
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "common.cuh"
#include "kernels.cuh"

static inline double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// Tracking-loss recovery (ll_mapper_set_recovery; DESIGN.md §4.3.2): the detection state, the attempt's own buffers (allocated when it is
// turned on), the step log and what the last attempt passed to the search.
struct Recovery {
  bool on = false;
  ll_recovery_cfg cfg;
  int state = LL_TRACKING, bad = 0;   // bad: consecutive bad steps
  bool field_valid = false;           // the field belongs to the map as it is in this loss episode
  ll_reloc_field* field = nullptr;
  ll_map* whole = nullptr;            // mode 1: the whole map, rebuilt in place once per episode
  DevBuf buf;                         // the step's features and the score points of each class (RecoveryLayout)
  EventLog<ll_recovery_step> log;
  ll_recovery_step* cur = nullptr;    // the current step's entry
  // the last attempt's inputs (the parity hook): host copies of the rotations and cfgs, the device features and score points in buf
  bool have_last = false;
  std::vector<double> rot_c, rot_f;
  ll_reloc_cfg coarse; ll_reloc_fine_cfg fine; ll_reg_state tmpl;
  size_t n_last[4] = {0, 0, 0, 0};
};
// buf: a step's features (corners then surfaces, scan frame), the score points of each class, their counts
struct RecoveryLayout {
  float4* feat; float4* score[2]; int* cnt;
  void layout(Carve& k, size_t n) { feat = k.take<float4>(n); score[0] = k.take<float4>(n); score[1] = k.take<float4>(n); cnt = k.take<int>(2); }
};

struct ll_mapper {
  ll_ctx* ctx = nullptr;
  HistoryWindow his[2];         // per class (0 corner, 1 surface), as cells and the match map's trees
  std::vector<int> his_frame;   // the frame index of each window segment (both windows push and pop together); loop feedback reads it
  double last_his_add_q[4] = {1, 0, 0, 0}, last_his_add_t[3] = {0, 0, 0};   // m_last_his_add_q / _t (uninitialised members in the reference: defined as identity / 0)
  ll_mapper_config cfg;
  ll_cellmap* cells[2] = {nullptr, nullptr};
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
  Recovery rec;                // tracking-loss recovery (off unless ll_mapper_set_recovery turned it on)
  LoopClosure* lc = nullptr;   // loop closure (off unless ll_mapper_set_loop_closure turned it on)
};

// frame: the front end's device record and, per class, the gathered piece segments and the first VoxelGrid's outputs
struct FrameLayout {
  FrameDev* dev; float4* cls[2]; float4* mid[2];
  void layout(Carve& k, size_t cap) { dev = k.take<FrameDev>(1); for (int c = 0; c < 2; c++) { cls[c] = k.take<float4>(cap); mid[c] = k.take<float4>(cap); } }
};

// snap: the match-map snapshot (the two whole-map VoxelGrid outputs) and their counts
struct SnapLayout {
  float4* cls[2]; int* cnt;
  void layout(Carve& k, size_t mc, size_t ms) { cls[0] = k.take<float4>(mc + 1); cls[1] = k.take<float4>(ms + 1); cnt = k.take<int>(2); }
};
// work: a scan's features per class down-sampled and in the world frame, their counts and the pose
struct WorkLayout {
  float4* down[2]; float4* world[2]; int* cnt; double* pose;
  void layout(Carve& k, size_t n) { for (float4*& p : down) p = k.take<float4>(n); for (float4*& p : world) p = k.take<float4>(n); cnt = k.take<int>(2); pose = k.take<double>(7); }
};

// The mapper's per-class settings (0 corner, 1 surface): the leaf of the map side's VoxelGrids and the range of the mode-1 assembly.
static float class_leaf(const ll_mapper_config& cfg, int c) { return c ? cfg.plane_resolution : cfg.line_resolution; }
static float class_range(const ll_mapper_config& cfg, int c) { return c ? cfg.maximum_search_range_surface : cfg.maximum_search_range_corner; }

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
  if (S) for (ll_cellmap* cm : m->cells) LL_TRY(ll_cellmap_reserve(ctx, cm, S, F));
  // The two map-side arenas, each at the largest of its consumers.  Both: the append's VoxelGrid of a scan's features and the refresh's
  // whole-map VoxelGrid and index build, whose halves map_side_pair runs side by side (corner on stream2 / scratch2, surface on the context's
  // stream / scratch).  scratch alone: the registration's query sort and K10 hash set.
  size_t side = voxel_grid_bytes(F);
  if (R) side = std::max(side, std::max(voxel_grid_bytes((int)R), tree_scratch_bytes((int)R)));
  const size_t reg = std::max(query_sort_bytes(F, 1), layout_bytes([&](Carve& c) { l1_set_layout(c, F); }));
  LL_CUDA(ctx, ctx->scratch.reserve_floor(std::max(side, reg)));
  LL_CUDA(ctx, ctx->scratch2.reserve_floor(side));
  if (!R) return LL_OK;
  for (HistoryWindow& h : m->his) LL_TRY(h.reserve(ctx, R));
  SnapLayout sn; LL_CUDA(ctx, m->snap.reserve_floor(layout_bytes([&](Carve& c) { sn.layout(c, R, R); })));
  for (BucketTree& t : m->match_map->tree) LL_CUDA(ctx, t.storage.reserve_floor(tree_storage_bytes((int)R)));
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
  int st = LL_OK;
  for (int c = 0; c < 2 && st == LL_OK; c++) st = ll_cellmap_create(ctx, cfg->cell_resolution, cfg->threshold_cell_revisit, cfg->max_cells, &m->cells[c]);
  if (st != LL_OK) { ll_cellmap_release(m->cells[0]); delete m; return st; }
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
  for (ll_cellmap* cm : m->cells) ll_cellmap_release(cm);
  if (m->match_map) ll_map_release(m->match_map);
  m->work.release(); m->snap.release();
  for (HistoryWindow& h : m->his) h.release();
  for (FrontGraph& g : m->frame_graph) if (g.exec) cudaGraphExecDestroy(g.exec);
  m->frame[0].release(); m->frame[1].release(); m->frame_vg[0].release(); m->frame_vg[1].release();
  ll_reloc_field_release(m->rec.field); if (m->rec.whole) ll_map_release(m->rec.whole); m->rec.buf.release();
  loop_release(m->lc);
  delete m;
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

static int recovery_step(ll_mapper* m, int nc, int ns, const ll_reg_state& st, const ll_reg_result* out, bool* hold);

static MapperWindow mapper_window(ll_mapper* m) {
  return MapperWindow{{&m->his[0], &m->his[1]}, &m->his_frame, m->q_w_curr, m->t_w_curr, m->last_his_add_q, m->last_his_add_t, &m->map_dirty};
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
    size_t n[2] = {0, 0}; const ll_point* src[2] = {nullptr, nullptr}; int fov[2] = {0, 0};
    for (int c = 0; c < 2; c++) {
      if (m->cfg.matching_mode == 0) { n[c] = m->his[c].live(); src[c] = (const ll_point*)m->his[c].data(); }   // :518-531: the concatenation of the history window (the live range of the flat array)
      else LL_TRY(ll_cellmap_assemble(ctx, m->cells[c], m->q_w_curr, m->t_w_curr, class_range(m->cfg, c), m->cfg.maximum_in_fov_angle, class_leaf(m->cfg, c),
                                      m->cfg.down_sample_replace, nullptr, 0, &n[c], &fov[c], &src[c]));
    }
    SnapLayout sn; LL_CUDA(ctx, m->snap.carve([&](Carve& k) { sn.layout(k, n[0], n[1]); }));
    LL_TRY(map_side_pair(ctx, s, [&](int c, cudaStream_t cs, DevBuf& scr) -> int {   // the whole-map VoxelGrids (:533-537)
      if (n[c] > 0) return launch_voxel_grid(ctx, cs, scr, (const float4*)src[c], (int)n[c], nullptr, class_leaf(m->cfg, c), sn.cls[c], sn.cnt + c);
      LL_CUDA(ctx, cudaMemsetAsync(sn.cnt + c, 0, 4, cs)); return LL_OK;
    }));
    int hc[2] = {0, 0};
    LL_CUDA(ctx, cudaMemcpyAsync(hc, sn.cnt, 8, cudaMemcpyDeviceToHost, s));
    LL_CUDA(ctx, cudaStreamSynchronize(s));
    m->have_map = false;
    if (hc[0] > 0 && hc[1] > 0) {
      LL_TRY(ll_map_rebuild(ctx, m->match_map, sn.cls[0], (size_t)hc[0], sn.cls[1], (size_t)hc[1], LL_FMT_XYZI16, LL_DEVICE));   // buffers reused: no allocation per scan
      m->have_map = true;
    }                      // :544-545
    for (int c = 0; c < 2; c++) { m->snap_n[c] = hc[c]; m->fov[c] = fov[c]; }
    m->map_dirty = false;
  }
  if (stats) { stats->ms_refresh = (float)(now_ms() - tp); stats->map_corner = m->snap_n[0]; stats->map_surf = m->snap_n[1]; stats->cells_in_fov_corner = m->fov[0]; stats->cells_in_fov_surf = m->fov[1]; }
  WorkLayout wl; LL_CUDA(ctx, m->work.carve([&](Carve& c) { wl.layout(c, (size_t)(nc > ns ? nc : ns)); }));
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
  if (m->rec.on) {   // a bad step is held back (and, once lost, relocalized)
    bool hold = false;
    LL_TRY(recovery_step(m, nc, ns, st, out, &hold));
    if (hold) return LL_OK;
  }
  tp = now_ms();   // no map yet: the gate of :199 returns 1
  if (out->status == 0) return LL_OK;                                           // rejected: frame discarded (:1413-1416)
  // ---- new features to the world frame (:1422-1432), VoxelGrid (:1434-1437), cell maps (:1492-1493)
  double* h = ctx->pin->mapper_pose; for (int k = 0; k < 4; k++) h[k] = out->q_w_curr[k]; for (int k = 0; k < 3; k++) h[4 + k] = out->t_w_curr[k];
  double* d_pose = wl.pose;
  LL_CUDA(ctx, cudaMemcpyAsync(d_pose, h, 7 * sizeof(double), cudaMemcpyHostToDevice, s));
  const int n[2] = {nc, ns}; const float4* feat[2] = {A.feat, A.feat + nc};
  LL_TRY(map_side_pair(ctx, s, [&](int c, cudaStream_t cs, DevBuf& scr) -> int {
    if (n[c] <= 0) { LL_CUDA(ctx, cudaMemsetAsync(wl.cnt + c, 0, 4, cs)); return LL_OK; }
    LL_TRY(launch_transform(ctx, cs, d_pose, feat[c], n[c], wl.world[c]));
    return launch_voxel_grid(ctx, cs, scr, wl.world[c], n[c], nullptr, class_leaf(m->cfg, c), wl.down[c], wl.cnt + c);
  }));
  LL_CUDA(ctx, cudaMemcpyAsync(hc, wl.cnt, 8, cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  const double tr0 = now_ms();
  // history window (:1439-1478): r_diff / t_diff compare the pose adopted from the PREVIOUS scan (m_q_w_curr is only overwritten at :1498) with the
  // pose of the last addition; history_add_t_step = history_add_angle_step = 0 (:83-84)
  bool pushed = false;
  {
    const double* q = m->q_w_curr; const double* lq = m->last_his_add_q;
    double dot = fabs(q[0] * lq[0] + q[1] * lq[1] + q[2] * lq[2] + q[3] * lq[3]); if (dot > 1.0) dot = 1.0;
    const double r_diff = 2.0 * acos(dot) * 57.3;
    double t2 = 0; for (int k = 0; k < 3; k++) t2 += (m->t_w_curr[k] - m->last_his_add_t[k]) * (m->t_w_curr[k] - m->last_his_add_t[k]);
    const double t_diff = sqrt(t2);
    if ((int)m->his[0].segs.size() < m->cfg.maximum_history_size || t_diff > 0.0 || r_diff > 0.0 * 57.3) {
      for (int k = 0; k < 4; k++) m->last_his_add_q[k] = m->q_w_curr[k]; for (int k = 0; k < 3; k++) m->last_his_add_t[k] = m->t_w_curr[k];
      pushed = true;
      for (int c = 0; c < 2; c++) LL_TRY(m->his[c].push(ctx, wl.down[c], (size_t)hc[c]));
      m->his_frame.push_back(m->frame_index);
    }
    for (int c = 0; c < 2; c++)   // each window by its own segment count; the frame indices follow the corner window's
      if ((int)m->his[c].segs.size() > m->cfg.maximum_history_size) { m->his[c].pop_front(); if (c == 0) m->his_frame.erase(m->his_frame.begin()); }
  }
  double tcell[3] = {now_ms(), 0, 0};   // before the cell maps, after the corner's, after the surface's
  for (int c = 0; c < 2; c++) { LL_TRY(ll_cellmap_append(ctx, m->cells[c], wl.down[c], (size_t)hc[c], LL_FMT_XYZI16, LL_DEVICE)); tcell[c + 1] = now_ms(); }
  if (m->trace && now_ms() - tp > 10.0)   // LL_MAPPER_TRACE=1: where a slow append went (transform + VoxelGrid + sync | history | corner cells | surface cells)
    fprintf(stderr, "ll_mapper trace: frame %d append %.2f ms = features %.2f + history %.2f + cells %.2f + %.2f\n", m->frame_index, now_ms() - tp, tr0 - tp, tcell[0] - tr0, tcell[1] - tcell[0], tcell[2] - tcell[1]);
  m->map_dirty = true;                                                           // m_if_mapping_updated_* (:1490-1491)
  if (stats) { stats->appended_corner = hc[0]; stats->appended_surf = hc[1]; stats->ms_append = (float)(now_ms() - tp); }
  if (m->rec.on) m->rec.cur->appended = 1;
  for (int k = 0; k < 4; k++) m->q_w_curr[k] = out->q_w_curr[k]; for (int k = 0; k < 3; k++) m->t_w_curr[k] = out->t_w_curr[k];   // :1496-1505
  if (m->lc) LL_TRY(loop_step(ctx, m->lc, d_pose, pushed, m->frame_index, mapper_window(m)));   // :1523-1564
  return LL_OK;
}

}  // extern "C"

static int frame_arena(ll_mapper* m, int a, FrameArena* fa) {
  ll_ctx* ctx = m->ctx;
  const int cap = m->frame_pieces * ctx->cfg.max_scan_points;
  FrameLayout fl; LL_CUDA(ctx, m->frame[a].carve([&](Carve& c) { fl.layout(c, (size_t)cap); }));
  *fa = FrameArena{fl.dev, {fl.cls[0], fl.cls[1]}, {fl.mid[0], fl.mid[1]}, cap, {&m->frame_vg[0], &m->frame_vg[1]}, &m->frame_graph[a]};
  return LL_OK;
}

// ---------------------------------------------------------------------------------------------- the input loop
// ll_mapper_process_scans / _frames / _sweeps: the front end of input k + 1 is enqueued on the streams `fs` (ll_ctx::fe_stream) before the
// mapper step(s) of input k, so it runs under them.  Nothing the mapper step reads or writes is touched by the front end, whose results only
// reach the mapper through the copy into A.feat; the extractor's host bookkeeping advances in input order.  So a sequence gives the results of
// its inputs called one at a time.  ll_mapper_process_scan / _frame / _sweep are the loops of one input on the context's own streams
// (ll_ctx::own_front): their front end keeps the greatest priority, as every other call of the context, and nothing is enqueued ahead.
//
// A front end enqueued ahead of an input that then fails: it is drained (it reads the caller's inputs) and its host bookkeeping undone, so that
// the extractor stands where the one-by-one calls leave it.
//
// Host records are staged in stage_in: reserved for `points` records (max_scan_points, or a spin handle's max_points) before the first front
// end, because a reallocation (cudaFree) would synchronise the device in the middle of the sequence.
static int reserve_stage(ll_ctx* ctx, int fmt, int where, size_t points) {
  if (where != LL_HOST || fmt == LL_FMT_XYZI16) return LL_OK;
  const size_t rec = fmt == LL_FMT_PCL32 ? 32 : (size_t)ctx->layout.point_step;
  LL_CUDA(ctx, ctx->stage_in.reserve(points * rec));
  return LL_OK;
}

// Argument checks, before anything is enqueued or the extractor's bookkeeping moves: LL_ERR_INVALID for an unknown format or memory kind or a
// null cloud of points (n clouds), LL_ERR_CAPACITY for an input over max_scan_points.
static int check_clouds(ll_ctx* ctx, int fmt, int where, size_t n, const void* const* raws, const size_t* ns) {
  if ((fmt != LL_FMT_XYZI16 && fmt != LL_FMT_PCL32 && fmt != LL_FMT_STRIDED) || (where != LL_HOST && where != LL_DEVICE)) {
    ctx->set_error("unknown point format or memory kind"); return LL_ERR_INVALID;
  }
  for (size_t k = 0; k < n; k++) if (!raws[k] && ns[k]) { ctx->set_error("null cloud of " + std::to_string(ns[k]) + " points"); return LL_ERR_INVALID; }
  return LL_OK;
}
static int scans_check(ll_ctx* ctx, int n_scans, const void* const* raws, const size_t* ns, int fmt, int where) {
  LL_TRY(check_clouds(ctx, fmt, where, (size_t)n_scans, raws, ns));
  for (int k = 0; k < n_scans; k++) if (ns[k] > (size_t)ctx->cfg.max_scan_points) { ctx->set_error("scan " + std::to_string(k) + " larger than max_scan_points"); return LL_ERR_CAPACITY; }
  return LL_OK;
}
// Frames also give the pieces a frame is cut into and the entries it publishes; LL_ERR_INVALID for a bad odom_mode, pieces or cap.
static int frames_check(ll_mapper* m, int n_frames, int n_heads, const void* const* raws, const size_t* ns, int fmt, int where, int odom_mode, int cap,
                        int* pieces, int* publish) {
  ll_ctx* ctx = m->ctx;
  *pieces = m->cfg.reg.if_motion_deblur ? 1 : m->cfg.pipeline.pieces;   // laser_feature_extractor.hpp:305-309
  if (*pieces < 1 || *pieces > m->frame_pieces) { ctx->set_error("pieces must be 1 ... 16"); return LL_ERR_INVALID; }
  if (odom_mode != 0 && odom_mode != 1) { ctx->set_error("odom_mode must be 0 or 1"); return LL_ERR_INVALID; }
  *publish = odom_mode ? *pieces : 1;                                            // :385-388
  if (cap < *publish) { ctx->set_error("cap smaller than the pieces to publish"); return LL_ERR_INVALID; }
  LL_TRY(check_clouds(ctx, fmt, where, (size_t)n_frames * n_heads, raws, ns));
  for (int f = 0; f < n_frames; f++) {
    size_t total = 0; for (int h = 0; h < n_heads; h++) total += ns[(size_t)f * n_heads + h];
    if (total > (size_t)ctx->cfg.max_scan_points) { ctx->set_error("frame " + std::to_string(f) + " (all heads) larger than max_scan_points"); return LL_ERR_CAPACITY; }
  }
  return LL_OK;
}
// Sweeps: the spin handle must share the mapper's context; a sweep over the handle's max_points, or, with loop closure on, over the loop
// closure's per-step full cloud (max_scan_points: a sweep's whole kept cloud is one step's, and the kept points can only be fewer), is
// LL_ERR_CAPACITY before anything is enqueued.
static int sweeps_check(ll_mapper* m, ll_spin* spin, int n_sweeps, const void* const* raws, const size_t* ns, int fmt, int where) {
  ll_ctx* ctx = m->ctx;
  if (spin_ctx(spin) != ctx) { ctx->set_error("spin handle created on another context than the mapper"); return LL_ERR_INVALID; }
  LL_TRY(check_clouds(ctx, fmt, where, (size_t)n_sweeps, raws, ns));
  for (int k = 0; k < n_sweeps; k++) {
    if (ns[k] > spin_max_points(spin)) { ctx->set_error("sweep " + std::to_string(k) + " larger than the spin handle's max_points"); return LL_ERR_CAPACITY; }
    if (m->lc && ns[k] > loop_step_capacity(m->lc)) { ctx->set_error("sweep " + std::to_string(k) + " larger than max_scan_points with loop closure on"); return LL_ERR_CAPACITY; }
  }
  return LL_OK;
}

// One mapper step of an input: its features as the front end left them (nc corners at `corner`, nsf surfaces at `surf`), the largest time
// stamp of its full cloud, and whether the step runs.
struct FrontStep { const float4* corner; const float4* surf; int nc, nsf; double max_t; bool runs; };

// The front end of one kind of input as inputs_run drives it:
//   arenas          the copies of the buffers its results lie in: input k's front end fills copy k % arenas behind fe_free[k % arenas], the
//                   event of the last hand-over out of it (input k - arenas's);
//   max_points()    the records stage_in must hold for one input;
//   enqueue(k)      input k's front end on fs.main;
//   finish(k, &n)   once it has completed, its results read before the next front end is enqueued: the n steps it gives, step(k, 0 ... n - 1);
//   loop_cloud(k)   its full cloud(s) into the loop closure's input, before the next front end may overwrite them;
//   save / restore  the host bookkeeping around a front end enqueued ahead of an input that then fails.
// A scan: one step, which does not run when the scan is dropped (<= 5 petals and not whole_frame, laser_feature_extractor.hpp:287); its
// features in tmp_a / tmp_b, max_features refused by front_end_counts.
struct ScanFront {
  static constexpr int arenas = 1;
  ll_ctx* ctx; const FrontStreams& fs; const void* const* raws; const size_t* ns; int fmt, where; const double* stamps; const ll_pipeline_cfg* pc;
  FrontStep s; ExtractState saved;
  size_t max_points() const { return (size_t)ctx->cfg.max_scan_points; }
  int enqueue(int k) { return scan_front_end_enqueue(ctx, fs, raws[k], ns[k], fmt, where, stamps[k], pc); }
  int finish(int, int* n_steps) {
    int dropped = 0; *n_steps = 1;
    LL_TRY(front_end_counts(ctx, pc, &s.nc, &s.nsf, &dropped));
    s.corner = ctx->A.tmp_a; s.surf = ctx->A.tmp_b; s.max_t = (double)ctx->last_full_max_t; s.runs = !dropped;
    return LL_OK;
  }
  FrontStep step(int, int) const { return s; }
  int loop_cloud(LoopClosure* lc, int) { return loop_scan_cloud(ctx, lc, pc); }   // the full cloud, compacted again from the extractor's state
  void save() { saved = ctx->ex; }
  void restore() { ctx->ex = saved; }
};
// A sweep: the spin handle's front end and the mapping node's VoxelGrids (spin_sweep_enqueue).  One step, which always runs: every sweep registers.
struct SweepFront {
  static constexpr int arenas = 1;
  ll_ctx* ctx; ll_spin* spin; const FrontStreams& fs; const void* const* raws; const size_t* ns; int fmt, where; const ll_pipeline_cfg* pc;
  FrontStep s;
  size_t max_points() const { return spin_max_points(spin); }
  int enqueue(int k) { return spin_sweep_enqueue(spin, fs, raws[k], ns[k], fmt, where, pc); }
  int finish(int k, int* n_steps) {
    float max_t = 0.f; *n_steps = 1;
    spin_sweep_finish(spin, ns[k], &s.corner, &s.nc, &s.surf, &s.nsf, &max_t);
    s.max_t = (double)max_t; s.runs = true;
    return LL_OK;
  }
  FrontStep step(int, int) const { return s; }
  int loop_cloud(LoopClosure* lc, int) { int n = 0; const int* d_n = nullptr; const float4* full = spin_full_cloud(spin, &n, &d_n); return loop_sweep_cloud(ctx, lc, full, n, d_n); }
  void save() {}
  void restore() { spin_forget(spin); }
};
// A frame: the piecewise front end (every head, every piece, one host read) into arena k & 1, so that frame k + 1's fills the other while frame
// k's pieces are still read out.  One step per published piece, none when no head is live (laser_feature_extractor.hpp:287, every head).
struct FrameFront {
  static constexpr int arenas = 2;
  ll_ctx* ctx; const FrontStreams& fs; int n_heads; const void* const* raws; const size_t* ns; int fmt, where; const double* stamps; const ll_pipeline_cfg* pc;
  int pieces = 0, publish = 0;
  FrameArena fa[2]; FrameOut fo; ExtractState saved;
  size_t max_points() const { return (size_t)ctx->cfg.max_scan_points; }
  int enqueue(int k) { const size_t o = (size_t)k * n_heads; return frame_front_end(ctx, fs, fa[k & 1], n_heads, raws + o, ns + o, fmt, where, stamps + o, pieces, pc); }
  int finish(int, int* n_steps) { fo = ctx->pin->frame; *n_steps = fo.heads_live != 0 ? publish : 0; return LL_OK; }
  FrontStep step(int k, int i) const {
    const int c0 = i ? fo.out_end[0][i - 1] : 0, s0 = i ? fo.out_end[1][i - 1] : 0;
    return {fa[k & 1].cls[0] + c0, fa[k & 1].cls[1] + s0, fo.out_end[0][i] - c0, fo.out_end[1][i] - s0, (double)ll_ord2f(fo.tmax[i]), true};
  }
  int loop_cloud(LoopClosure* lc, int k) { return loop_frame_clouds(ctx, lc, fa[k & 1].dev, ns + (size_t)k * n_heads, n_heads, publish); }
  void save() { saved = ctx->ex; }
  void restore() { ctx->ex = saved; }
};

// Input k: the front end, then per step i its features into A.feat and mapper_step, the entry at out / stats [k * cap + i].  A step that is
// refused or fails ends the sequence; a rejected step leaves the pose as it was, and the next step continues from there.
template <typename Front>
static int inputs_run(ll_mapper* m, Front& fe, int n_inputs, ll_reg_result* out, ll_mapper_stats* stats, int cap, int* n_pieces, int* done) {
  ll_ctx* ctx = m->ctx;
  const FrontStreams& fs = fe.fs;
  LL_TRY(reserve_stage(ctx, fe.fmt, fe.where, fe.max_points()));
  auto enqueue = [&](int k) -> int {
    LL_CUDA(ctx, cudaStreamWaitEvent(fs.main, ctx->sev.fe_free[k % Front::arenas], 0));
    LL_TRY(fe.enqueue(k));
    LL_CUDA(ctx, cudaEventRecord(ctx->sev.fe_ready, fs.main));
    return LL_OK;
  };
  bool ahead = false;
  const int st = [&]() -> int {
    double t = now_ms();
    LL_TRY(enqueue(0));
    float ms_enqueue = (float)(now_ms() - t);
    for (int k = 0; k < n_inputs; k++) {
      ahead = false;
      t = now_ms();
      LL_CUDA(ctx, cudaEventSynchronize(ctx->sev.fe_ready));
      int n_steps = 0;
      LL_TRY(fe.finish(k, &n_steps));
      const float ms_front_end = ms_enqueue + (float)(now_ms() - t);
      // the next front end goes under this input's steps unless one of them will stop the sequence at features_fit
      bool next = k + 1 < n_inputs;
      for (int i = 0; i < n_steps; i++) { const FrontStep s = fe.step(k, i); next = next && (!s.runs || s.nc + s.nsf <= ctx->cfg.max_features); }
      auto enqueue_next = [&]() -> int {
        if (!next) return LL_OK;
        fe.save(); ahead = true;
        const double t1 = now_ms();
        LL_TRY(enqueue(k + 1));
        ms_enqueue = (float)(now_ms() - t1);
        return LL_OK;
      };
      // Two arenas: the full clouds lie outside them (tmp_c), where the next front end overwrites them whichever arena it fills, so they are
      // captured ahead of the steps, behind an event of their own that the next front end waits on.  One arena: after the step's hand-over,
      // whose fe_free guards both.
      if (Front::arenas == 2 && m->lc && n_steps > 0) {
        LL_TRY(fe.loop_cloud(m->lc, k));
        LL_CUDA(ctx, cudaEventRecord(ctx->sev.fe_free[(k + 1) % Front::arenas], ctx->stream));
      }
      if (n_steps == 0) LL_TRY(enqueue_next());
      for (int i = 0; i < n_steps; i++) {
        const FrontStep s = fe.step(k, i);
        ll_reg_result* o = out + (size_t)k * cap + i;
        ll_mapper_stats* ps = stats ? stats + (size_t)k * cap + i : nullptr;
        if (ps) { memset(ps, 0, sizeof(*ps)); ps->n_corner = s.nc; ps->n_surf = s.nsf; ps->ms_front_end = i == 0 ? ms_front_end : 0.f; }
        out_init(m, o);
        if (s.runs) {
          LL_TRY(features_fit(ctx, s.nc, s.nsf));
          LL_TRY(features_hand_over(ctx, ctx->stream, s.corner, s.nc, s.surf, s.nsf));
          if (Front::arenas == 1 && m->lc) LL_TRY(fe.loop_cloud(m->lc, k));
        }
        if (i == n_steps - 1) LL_CUDA(ctx, cudaEventRecord(ctx->sev.fe_free[k % Front::arenas], ctx->stream));
        if (i == 0) LL_TRY(enqueue_next());
        if (m->lc) loop_select_piece(m->lc, i);
        if (s.runs) LL_TRY(mapper_step(m, s.nc, s.nsf, s.max_t, o, ps));
        if (n_pieces) n_pieces[k] = i + 1;
      }
      *done = k + 1;
    }
    return LL_OK;
  }();
  if (st != LL_OK) {
    for (cudaStream_t s : {fs.main, fs.corner, fs.petals}) cudaStreamSynchronize(s);
    if (ahead) fe.restore();
  }
  return st;
}

static int run_scans(ll_mapper* m, const FrontStreams& fs, int n_scans, const void* const* raws, const size_t* ns, int fmt, int where, const double* stamps,
                     ll_reg_result* out, ll_mapper_stats* stats, int* done) {
  LL_TRY(scans_check(m->ctx, n_scans, raws, ns, fmt, where));
  ScanFront fe{m->ctx, fs, raws, ns, fmt, where, stamps, &m->cfg.pipeline};
  return inputs_run(m, fe, n_scans, out, stats, 1, nullptr, done);
}
static int run_frames(ll_mapper* m, const FrontStreams& fs, int n_frames, int n_heads, const void* const* raws, const size_t* ns, int fmt, int where,
                      const double* stamps, int odom_mode, ll_reg_result* out, ll_mapper_stats* stats, int cap, int* n_pieces, int* done) {
  FrameFront fe{m->ctx, fs, n_heads, raws, ns, fmt, where, stamps, &m->cfg.pipeline};
  LL_TRY(frames_check(m, n_frames, n_heads, raws, ns, fmt, where, odom_mode, cap, &fe.pieces, &fe.publish));
  for (int f = 0; f < n_frames; f++) n_pieces[f] = 0;
  LL_TRY(frame_arena(m, 0, &fe.fa[0])); LL_TRY(frame_arena(m, 1, &fe.fa[1]));
  return inputs_run(m, fe, n_frames, out, stats, cap, n_pieces, done);
}
static int run_sweeps(ll_mapper* m, ll_spin* spin, const FrontStreams& fs, int n_sweeps, const void* const* raws, const size_t* ns, int fmt, int where,
                      ll_reg_result* out, ll_mapper_stats* stats, int* done) {
  LL_TRY(sweeps_check(m, spin, n_sweeps, raws, ns, fmt, where));
  SweepFront fe{m->ctx, spin, fs, raws, ns, fmt, where, &m->cfg.pipeline};
  return inputs_run(m, fe, n_sweeps, out, stats, 1, nullptr, done);
}

extern "C" int ll_mapper_process_scan(ll_mapper* m, const void* raw, size_t n, int fmt, int where, double stamp, ll_reg_result* out, ll_mapper_stats* stats) {
  if (!m || !out) return LL_ERR_INVALID;
  ll_ctx* ctx = m->ctx; cudaSetDevice(ctx->device);
  int done = 0;
  return run_scans(m, ctx->own_front(), 1, &raw, &n, fmt, where, &stamp, out, stats, &done);
}

extern "C" int ll_mapper_process_scans(ll_mapper* m, int n_scans, const void* const* raws, const size_t* ns, int fmt, int where, const double* stamps,
                                       ll_reg_result* out, ll_mapper_stats* stats, int* n_scans_done) {
  if (n_scans_done) *n_scans_done = 0;
  if (!m || !out || !raws || !ns || !stamps || !n_scans_done || n_scans < 1) return LL_ERR_INVALID;
  ll_ctx* ctx = m->ctx; cudaSetDevice(ctx->device);
  return run_scans(m, ctx->pipe_front(), n_scans, raws, ns, fmt, where, stamps, out, stats, n_scans_done);
}

extern "C" int ll_mapper_process_frame(ll_mapper* m, int n_heads, const void* const* raws, const size_t* ns, int fmt, int where, const double* stamps,
                                       int odom_mode, ll_reg_result* out, ll_mapper_stats* stats, int cap, int* n_pieces) {
  if (!m || !out || !raws || !ns || !stamps || !n_pieces || n_heads < 1 || n_heads > LL_MAX_HEADS) return LL_ERR_INVALID;
  *n_pieces = 0;
  ll_ctx* ctx = m->ctx; cudaSetDevice(ctx->device);
  int done = 0;
  return run_frames(m, ctx->own_front(), 1, n_heads, raws, ns, fmt, where, stamps, odom_mode, out, stats, cap, n_pieces, &done);
}

extern "C" int ll_mapper_process_frames(ll_mapper* m, int n_frames, int n_heads, const void* const* raws, const size_t* ns, int fmt, int where,
                                        const double* stamps, int odom_mode, ll_reg_result* out, ll_mapper_stats* stats, int cap, int* n_pieces, int* n_frames_done) {
  if (n_frames_done) *n_frames_done = 0;
  if (!m || !out || !raws || !ns || !stamps || !n_pieces || !n_frames_done || n_frames < 1 || n_heads < 1 || n_heads > LL_MAX_HEADS) return LL_ERR_INVALID;
  ll_ctx* ctx = m->ctx; cudaSetDevice(ctx->device);
  return run_frames(m, ctx->pipe_front(), n_frames, n_heads, raws, ns, fmt, where, stamps, odom_mode, out, stats, cap, n_pieces, n_frames_done);
}

extern "C" int ll_mapper_process_sweep(ll_mapper* m, ll_spin* spin, const void* raw, size_t n, int fmt, int where, ll_reg_result* out, ll_mapper_stats* stats) {
  if (!m || !spin || !out) return LL_ERR_INVALID;
  ll_ctx* ctx = m->ctx; cudaSetDevice(ctx->device);
  int done = 0;
  return run_sweeps(m, spin, ctx->own_front(), 1, &raw, &n, fmt, where, out, stats, &done);
}

extern "C" int ll_mapper_process_sweeps(ll_mapper* m, ll_spin* spin, int n_sweeps, const void* const* raws, const size_t* ns, int fmt, int where,
                                        ll_reg_result* out, ll_mapper_stats* stats, int* n_sweeps_done) {
  if (n_sweeps_done) *n_sweeps_done = 0;
  if (!m || !spin || !out || !raws || !ns || !n_sweeps_done || n_sweeps < 1) return LL_ERR_INVALID;
  ll_ctx* ctx = m->ctx; cudaSetDevice(ctx->device);
  return run_sweeps(m, spin, ctx->pipe_front(), n_sweeps, raws, ns, fmt, where, out, stats, n_sweeps_done);
}

// ---------------------------------------------------------------------------------------------- checkpoint
// The image (format: include/loamlivox_b200.h) holds what the next steps read: the config, the scalars, the history window, the snapshot
// the kNN index was built from (the index's own copy of its input, BucketTree::src), both cell maps and the extractor's time bookkeeping.
// One host validator serves ll_mapper_image_info and ll_mapper_load, before anything touches the device.
namespace {

const ImageKind MAPPER_IMAGE{LL_MAPPER_IMAGE_MAGIC, "mapper", LL_MAPPER_IMAGE_VERSION, LL_MAPPER_IMAGE_VERSION, sizeof(ll_mapper_config), "ll_mapper_config",
                             LL_IMAGE_SECTIONS};
const size_t SNAP_HEAD = 8;   // the fixed part of a snapshot section

struct ImageView {   // a validated image
  ll_mapper_image_header h; ll_mapper_config cfg; ll_mapper_image_scalars sc;
  HistoryView his[2];
  struct { int64_t n = 0; const uint8_t* pts = nullptr; } snap[2];
  CellsView cells[2];
};

// LL_OK, or the code and what is wrong.  cfg: the caller's config for a load (NULL: the image's).
int image_validate(const void* image, size_t bytes, const ll_mapper_config* cfg, ImageView* v, std::string* err) {
  auto fail = [&](const char* msg, int code = LL_ERR_INVALID) { if (err) *err = msg; return code; };
  const uint8_t* b = (const uint8_t*)image;
  LL_TRY(image_structure(image, bytes, MAPPER_IMAGE, v->h.section, err));
  memcpy(&v->h, b, sizeof(v->h));
  auto sec = [&](int k) { return b + v->h.section[k].offset; };
  auto len = [&](int k) { return (uint64_t)v->h.section[k].length; };
  // config: ll_mapper_create's checks and a matching mode the mapper knows
  if (len(LL_IMAGE_CONFIG) != sizeof(ll_mapper_config)) return fail("config section length");
  memcpy(&v->cfg, sec(LL_IMAGE_CONFIG), sizeof(v->cfg));
  if (!(v->cfg.cell_resolution > 0.f) || v->cfg.threshold_cell_revisit < 1) return fail("config: cell_resolution must be > 0 and threshold_cell_revisit >= 1");
  if (v->cfg.max_cells > MAX_CELLS) return fail("config: max_cells must be <= 2^29");
  if (v->cfg.matching_mode != 0 && v->cfg.matching_mode != 1) return fail("config: matching_mode must be 0 or 1");
  // scalars
  if (len(LL_IMAGE_SCALARS) != sizeof(ll_mapper_image_scalars)) return fail("scalars section length");
  memcpy(&v->sc, sec(LL_IMAGE_SCALARS), sizeof(v->sc));
  const ll_mapper_image_scalars& sc = v->sc;
  const double times[] = {sc.last_time_stamp, sc.first_receive_time, sc.current_time, sc.last_maximum_time_stamp};
  if (!finite_d(times, 4) || !finite_d(sc.q_w_curr, 4) || !finite_d(sc.t_w_curr, 3) || !finite_d(sc.last_his_add_q, 4) || !finite_d(sc.last_his_add_t, 3))
    return fail("non-finite pose or time stamp");
  if (sc.frame_index < 0 || (sc.map_dirty != 0 && sc.map_dirty != 1) || (sc.have_map != 0 && sc.have_map != 1) || sc.reserved != 0 ||
      sc.snap_n[0] < 0 || sc.snap_n[1] < 0 || sc.fov[0] < 0 || sc.fov[1] < 0)
    return fail("scalars out of range");
  if (sc.have_map && (sc.snap_n[0] == 0 || sc.snap_n[1] == 0)) return fail("have_map with an empty snapshot");
  for (int c = 0; c < 2; c++) {
    if (const char* e = history_section(sec(LL_IMAGE_HISTORY_CORNER + c), len(LL_IMAGE_HISTORY_CORNER + c), true, &v->his[c])) return fail(e);
    // snapshot: as many points as snap_n when the index exists, none otherwise
    {
      const uint8_t* p = sec(LL_IMAGE_SNAPSHOT_CORNER + c); const uint64_t L = len(LL_IMAGE_SNAPSHOT_CORNER + c);
      if (L < SNAP_HEAD) return fail("snapshot section shorter than its count");
      const int64_t n = img_get<int64_t>(p);
      if (n < 0 || (uint64_t)n > (L - SNAP_HEAD) / 16 || SNAP_HEAD + 16 * (uint64_t)n != L) return fail("snapshot count disagrees with the section length");
      if (n != (sc.have_map ? sc.snap_n[c] : 0)) return fail("snapshot disagrees with have_map / snap_n");
      for (int64_t k = 0; k < n; k++) if (!finite_xyz(p + SNAP_HEAD + 16 * k)) return fail("non-finite snapshot point");
      v->snap[c].n = n; v->snap[c].pts = p + SNAP_HEAD;
    }
    if (const char* e = cells_section(sec(LL_IMAGE_CELLS_CORNER + c), len(LL_IMAGE_CELLS_CORNER + c), false, &v->cells[c])) return fail(e);
  }
  // the caller's config: the image's but for the buffer sizes
  if (cfg) {
    ll_mapper_config x = *cfg;
    x.max_cells = v->cfg.max_cells; x.reserve_map_points = v->cfg.reserve_map_points; x.reserve_store_points = v->cfg.reserve_store_points;
    if (memcmp(&x, &v->cfg, sizeof(x)) != 0) return fail("cfg differs from the image's config in a field other than max_cells, reserve_map_points, reserve_store_points");
  }
  const int max_cells = cfg ? cfg->max_cells : v->cfg.max_cells;
  for (int c = 0; c < 2; c++) {
    if (const char* e = load_capacity(v->cells[c], v->his[c], &max_cells)) return fail(e, LL_ERR_CAPACITY);
    if (v->snap[c].n > INT32_MAX) return fail("more points than a map holds", LL_ERR_CAPACITY);
  }
  return LL_OK;
}

// The validated image's state into a mapper just created with its effective config.
int mapper_restore(ll_mapper* m, const ImageView& v) {
  ll_ctx* ctx = m->ctx;
  cudaStream_t s = ctx->stream;
  const ll_mapper_image_scalars& sc = v.sc;
  m->frame_index = sc.frame_index; m->last_time_stamp = sc.last_time_stamp;
  for (int k = 0; k < 4; k++) { m->q_w_curr[k] = sc.q_w_curr[k]; m->last_his_add_q[k] = sc.last_his_add_q[k]; }
  for (int k = 0; k < 3; k++) { m->t_w_curr[k] = sc.t_w_curr[k]; m->last_his_add_t[k] = sc.last_his_add_t[k]; }
  m->map_dirty = sc.map_dirty != 0;
  for (int c = 0; c < 2; c++) { m->snap_n[c] = sc.snap_n[c]; m->fov[c] = sc.fov[c]; }
  ctx->ex.first_receive_time = sc.first_receive_time; ctx->ex.current_time = sc.current_time; ctx->ex.last_maximum_time_stamp = sc.last_maximum_time_stamp;
  for (int c = 0; c < 2; c++) LL_TRY(history_restore(ctx, m->his[c], v.his[c]));
  // The image does not hold the segments' frame indices (a version-3 loop image does, and its load sets them).  Here they are numbered up to
  // the frame index: ascending and no later than it, so before any keyframe a loop closure set on this mapper can close, whose correction at
  // such a step is the identity.
  m->his_frame.resize((size_t)v.his[0].n_seg);
  for (size_t k = 0; k < m->his_frame.size(); k++) m->his_frame[k] = sc.frame_index - (int)(m->his_frame.size() - 1 - k);
  for (int c = 0; c < 2; c++) LL_TRY(cells_restore(ctx, m->cells[c], v.cells[c], false));
  // the snapshot and its index (the build is deterministic: the kNN answers are the saved mapper's)
  m->have_map = false;
  if (sc.have_map) {
    const size_t n[2] = {(size_t)v.snap[0].n, (size_t)v.snap[1].n};
    SnapLayout sn; LL_CUDA(ctx, m->snap.carve([&](Carve& k) { sn.layout(k, n[0], n[1]); }));
    for (int c = 0; c < 2; c++) LL_CUDA(ctx, cudaMemcpyAsync(sn.cls[c], v.snap[c].pts, n[c] * 16, cudaMemcpyHostToDevice, s));
    LL_TRY(ll_map_rebuild(ctx, m->match_map, sn.cls[0], n[0], sn.cls[1], n[1], LL_FMT_XYZI16, LL_DEVICE));
    m->have_map = true;
  }
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  return LL_OK;
}

}  // namespace

extern "C" int ll_mapper_save(ll_mapper* m, void* image, size_t cap, size_t* bytes) {
  if (!m || !bytes) return LL_ERR_INVALID;
  ll_ctx* ctx = m->ctx; cudaSetDevice(ctx->device);
  cudaStream_t s = ctx->stream;
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  int64_t n_snap[2]; CellsView cells[2];
  for (int c = 0; c < 2; c++) {
    n_snap[c] = m->have_map ? m->match_map->tree[c].n_src : 0;
    if (m->have_map && n_snap[c] != m->snap_n[c]) { ctx->set_error("match-map index and snapshot disagree"); return LL_ERR_INVALID; }
    int nc = 0, live = 0;
    LL_TRY(cm_count(ctx, m->cells[c], &nc, &live, &cells[c].frame_idx, &cells[c].n_oor));
    cells[c].n_cells = nc; cells[c].n_pts = live;
  }
  const uint64_t len[LL_IMAGE_SECTIONS] = {sizeof(ll_mapper_config), sizeof(ll_mapper_image_scalars), history_bytes(m->his[0]), history_bytes(m->his[1]),
                                           SNAP_HEAD + 16 * (uint64_t)n_snap[0], SNAP_HEAD + 16 * (uint64_t)n_snap[1], cells_bytes(cells[0], false),
                                           cells_bytes(cells[1], false)};
  ll_mapper_image_header h;
  const size_t total = image_header(MAPPER_IMAGE, LL_MAPPER_IMAGE_VERSION, len, &h);
  *bytes = total;
  if (!image) return LL_OK;
  if (cap < total) { ctx->set_error("image buffer smaller than the image (query the size with image = NULL)"); return LL_ERR_CAPACITY; }
  uint8_t* b = (uint8_t*)image;
  auto at = [&](int k) { return b + h.section[k].offset; };
  memcpy(b, &h, sizeof(h));
  memcpy(at(LL_IMAGE_CONFIG), &m->cfg, sizeof(m->cfg));
  ll_mapper_image_scalars sc; memset(&sc, 0, sizeof(sc));
  sc.frame_index = m->frame_index; sc.map_dirty = m->map_dirty ? 1 : 0; sc.have_map = m->have_map ? 1 : 0;
  for (int c = 0; c < 2; c++) { sc.snap_n[c] = m->snap_n[c]; sc.fov[c] = m->fov[c]; }
  sc.last_time_stamp = m->last_time_stamp;
  for (int k = 0; k < 4; k++) { sc.q_w_curr[k] = m->q_w_curr[k]; sc.last_his_add_q[k] = m->last_his_add_q[k]; }
  for (int k = 0; k < 3; k++) { sc.t_w_curr[k] = m->t_w_curr[k]; sc.last_his_add_t[k] = m->last_his_add_t[k]; }
  sc.first_receive_time = ctx->ex.first_receive_time; sc.current_time = ctx->ex.current_time; sc.last_maximum_time_stamp = ctx->ex.last_maximum_time_stamp;
  memcpy(at(LL_IMAGE_SCALARS), &sc, sizeof(sc));
  for (int c = 0; c < 2; c++) {
    LL_TRY(history_write(ctx, m->his[c], at(LL_IMAGE_HISTORY_CORNER + c)));
    uint8_t* p = at(LL_IMAGE_SNAPSHOT_CORNER + c);
    img_put<int64_t>(p, n_snap[c]);
    if (n_snap[c]) LL_CUDA(ctx, cudaMemcpyAsync(p + SNAP_HEAD, m->match_map->tree[c].src, (size_t)n_snap[c] * 16, cudaMemcpyDeviceToHost, s));
    LL_TRY(cells_write(ctx, m->cells[c], cells[c], at(LL_IMAGE_CELLS_CORNER + c)));
  }
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  return LL_OK;
}

extern "C" int ll_mapper_load(ll_ctx* ctx, const void* image, size_t bytes, const ll_mapper_config* cfg, ll_mapper** out) {
  if (!ctx || !out) return LL_ERR_INVALID;
  *out = nullptr;
  ImageView v; std::string err;
  const int st = image_validate(image, bytes, cfg, &v, &err);
  if (st != LL_OK) { ctx->set_error("mapper image refused: " + err); return st; }
  cudaSetDevice(ctx->device);
  ll_mapper* m = nullptr;
  LL_TRY(ll_mapper_create(ctx, cfg ? cfg : &v.cfg, &m));
  const int rs = mapper_restore(m, v);
  if (rs != LL_OK) { ll_mapper_release(m); return rs; }
  // The buffer sizes of cfg sized this mapper's allocations (they are read at creation only); its images keep the stream's config, so that
  // load-then-save reproduces an image whatever sizes the load chose.
  m->cfg = v.cfg;
  *out = m;
  return LL_OK;
}

extern "C" int ll_mapper_image_info(const void* image, size_t bytes, ll_image_info* info) {
  if (!info) return LL_ERR_INVALID;
  ImageView v;
  LL_TRY(image_validate(image, bytes, nullptr, &v, nullptr));
  memset(info, 0, sizeof(*info));
  info->bytes = bytes; info->version = v.h.version; info->matching_mode = v.cfg.matching_mode;
  info->frame_index = v.sc.frame_index; info->have_map = v.sc.have_map; info->map_dirty = v.sc.map_dirty;
  for (int c = 0; c < 2; c++) {
    info->history_points[c] = v.his[c].n_pts; info->history_segments[c] = (int32_t)v.his[c].n_seg; info->snapshot_points[c] = v.snap[c].n;
    info->cells[c] = v.cells[c].n_cells; info->cell_points[c] = v.cells[c].n_pts; info->cell_frame_idx[c] = v.cells[c].frame_idx;
  }
  return LL_OK;
}

// ---------------------------------------------------------------------------------------------- relocalization glue
// The whole map as a new ll_map: the clouds (mode 0: the live history window; mode 1: every live point of each cell map in store order) into
// the context's feat_buf, their VoxelGrids at the line / plane resolution, and an index built in place.  Nothing of the mapper is written.
// The whole map's two VoxelGrid outputs in the context's feat_buf: vg[c], hc[c] points (on the device once this returns).
static int whole_map_clouds(ll_mapper* m, float4* vg[2], int hc[2]) {
  ll_ctx* ctx = m->ctx;
  cudaStream_t s = ctx->stream;
  size_t n[2] = {0, 0};
  if (m->cfg.matching_mode == 0) {
    for (int c = 0; c < 2; c++) n[c] = m->his[c].live();
  } else {
    for (int c = 0; c < 2; c++) { int cells = 0, live = 0, fi = 0, oor = 0; LL_TRY(cm_count(ctx, m->cells[c], &cells, &live, &fi, &oor)); n[c] = (size_t)live; }
  }
  if (n[0] == 0 || n[1] == 0) { ctx->set_error("the mapper has no map yet (a class is empty)"); return LL_ERR_INVALID; }
  float4* in[2] = {nullptr, nullptr}; int* d_cnt;
  LL_CUDA(ctx, ctx->feat_buf.carve([&](Carve& c) {
    if (m->cfg.matching_mode == 1) { in[0] = c.take<float4>(n[0]); in[1] = c.take<float4>(n[1]); }
    vg[0] = c.take<float4>(n[0]); vg[1] = c.take<float4>(n[1]); d_cnt = c.take<int>(2);
  }));
  for (int c = 0; c < 2; c++) {
    const float4* src = m->his[c].data();
    if (m->cfg.matching_mode == 1) { LL_TRY(cm_live_points(ctx, m->cells[c], (int)n[c], in[c])); src = in[c]; }
    LL_TRY(launch_voxel_grid(ctx, s, ctx->scratch, src, (int)n[c], nullptr, class_leaf(m->cfg, c), vg[c], d_cnt + c));
  }
  LL_CUDA(ctx, cudaMemcpyAsync(hc, d_cnt, 2 * sizeof(int), cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  return LL_OK;
}

extern "C" int ll_mapper_whole_map(ll_mapper* m, ll_map** out) {
  if (!m || !out) return LL_ERR_INVALID;
  *out = nullptr;
  ll_ctx* ctx = m->ctx; cudaSetDevice(ctx->device);
  cudaStream_t s = ctx->stream;
  float4* vg[2]; int hc[2] = {0, 0};
  LL_TRY(whole_map_clouds(m, vg, hc));
  ll_map* map = nullptr;
  LL_TRY(ll_map_build(ctx, vg[0], (size_t)hc[0], vg[1], (size_t)hc[1], LL_FMT_XYZI16, LL_DEVICE, &map));
  if (cudaStreamSynchronize(s) != cudaSuccess) { ll_map_release(map); ctx->set_error("whole-map index build failed"); return LL_ERR_CUDA; }
  *out = map;
  return LL_OK;
}

// ll_mapper_set_pose after its checks (also the adoption of a relocalized pose).
static void mapper_set_pose(ll_mapper* m, const double q_wxyz[4], const double t[3]) {
  if (memcmp(q_wxyz, m->q_w_curr, sizeof(m->q_w_curr)) == 0 && memcmp(t, m->t_w_curr, sizeof(m->t_w_curr)) == 0) return;
  for (int k = 0; k < 4; k++) m->q_w_curr[k] = q_wxyz[k];
  for (int k = 0; k < 3; k++) m->t_w_curr[k] = t[k];
  if (m->cfg.matching_mode == 1) m->map_dirty = true;   // the assembly of mode 1 is around the pose
}

extern "C" int ll_mapper_set_pose(ll_mapper* m, const double q_wxyz[4], const double t[3]) {
  if (!m || !q_wxyz || !t) return LL_ERR_INVALID;
  for (int k = 0; k < 4; k++) if (!std::isfinite(q_wxyz[k])) return LL_ERR_INVALID;
  for (int k = 0; k < 3; k++) if (!std::isfinite(t[k])) return LL_ERR_INVALID;
  mapper_set_pose(m, q_wxyz, t);
  return LL_OK;
}

// ---------------------------------------------------------------------------------------------- tracking-loss recovery
// DESIGN.md §4.3.2.  Detection runs on the host from the step's ll_reg_result; the attempt is the library's own path: the whole map, the field
// build shared with ll_reloc_field_build, the VoxelGrid launcher for the score points and ll_relocalize_field on device inputs.
namespace {

void yaw_quat(double deg, double* q) { const double a = deg * (M_PI / 180.0) * 0.5; q[0] = cos(a); q[1] = 0; q[2] = 0; q[3] = sin(a); }
int coarse_yaws(const ll_recovery_cfg& c) { return (int)std::lround(360.0 / c.yaw_step_deg); }
int fine_yaws(const ll_recovery_cfg& c) { return 2 * (int)std::floor(0.5 * c.yaw_step_deg / c.fine_yaw_step_deg + 1e-9) + 1; }
int fine_nt(const ll_recovery_cfg& c) { return 2 * (int)std::floor(c.fine_t_half * c.t_step / c.fine_t_step + 1e-9) + 1; }

const char* recovery_cfg_error(const ll_recovery_cfg& c) {
  auto pos = [](double x) { return std::isfinite(x) && x > 0.0; };
  auto nonneg = [](double x) { return std::isfinite(x) && x >= 0.0; };
  if (!nonneg(c.max_inlier_threshold)) return "max_inlier_threshold must be finite and >= 0";
  if (c.lost_after < 1) return "lost_after must be >= 1";
  if (c.trunc < 1 || c.trunc > 15) return "trunc must be 1 ... 15";
  if (!pos(c.res)) return "res must be finite and > 0";
  if (!pos(c.score_leaf)) return "score_leaf must be finite and > 0";
  if (!pos(c.yaw_step_deg) || c.yaw_step_deg > 360.0) return "yaw_step_deg must be in (0, 360]";
  if (!pos(c.t_step)) return "t_step must be finite and > 0";
  if (!nonneg(c.window_base) || !nonneg(c.window_growth)) return "window_base and window_growth must be finite and >= 0";
  if (c.max_candidates < 1 || c.max_candidates > LL_MAX_BATCH) return "max_candidates must be 1 ... LL_MAX_BATCH";
  if (c.max_hypotheses < 1 || c.max_hypotheses > (1 << 24)) return "max_hypotheses must be 1 ... 2^24";
  if (!pos(c.fine_yaw_step_deg) || !pos(c.fine_t_step) || !nonneg(c.fine_t_half)) return "fine steps must be finite and > 0, fine_t_half >= 0";
  if (!(c.min_verify_fraction >= 0.0 && c.min_verify_fraction <= 1.0)) return "min_verify_fraction must be 0 ... 1";
  if (c.reserve_field_voxels < 0 || c.reserve_field_voxels > (1ll << 30) || c.reserve_whole_map_points < 0 || c.reserve_whole_map_points > INT32_MAX)
    return "reservations must be >= 0 (field voxels <= 2^30, whole-map points <= 2^31 - 1)";
  if (coarse_yaws(c) > c.max_hypotheses) return "the yaw circle alone exceeds max_hypotheses";
  const double fine = (double)c.max_candidates * fine_yaws(c) * fine_nt(c) * fine_nt(c);
  if (fine > c.max_hypotheses) return "max_candidates x the fine hypotheses exceed max_hypotheses";
  return nullptr;
}

size_t buf_caps(ll_mapper* m) {   // the bytes held by every buffer an attempt may grow
  ll_ctx* ctx = m->ctx;
  size_t b = ctx->scratch.cap + ctx->scratch2.cap + ctx->feat_buf.cap + ctx->stage_in.cap + m->rec.buf.cap;
  if (m->rec.field) b += reloc_field_storage_cap(m->rec.field);
  if (m->rec.whole) for (const BucketTree& t : m->rec.whole->tree) b += t.storage.cap;
  return b;
}

// One class of the step's features through one VoxelGrid at the score leaf, the leaf doubled until the output fits LL_RELOC_MAX_SCORE_POINTS.
int score_points(ll_ctx* ctx, const float4* src, int n, float leaf, float4* dst, int* d_cnt, int* n_out, float* leaf_out) {
  *n_out = 0; *leaf_out = leaf;
  if (n <= 0) return LL_OK;
  for (;;) {
    LL_TRY(launch_voxel_grid(ctx, ctx->stream, ctx->scratch, src, n, nullptr, leaf, dst, d_cnt));
    int h = 0;
    LL_CUDA(ctx, cudaMemcpyAsync(&h, d_cnt, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *n_out = h; *leaf_out = leaf;
    if (h <= LL_RELOC_MAX_SCORE_POINTS) return LL_OK;
    leaf *= 2.f;
  }
}

}  // namespace

// The relocalization of one lost step (features nc + ns in A.feat, registration state st) into the log entry e; the pose is adopted when the
// choice passes the acceptance rule.
static int recovery_attempt(ll_mapper* m, int nc, int ns, const ll_reg_state& st, ll_recovery_step* e) {
  ll_ctx* ctx = m->ctx;
  Recovery& R = m->rec;
  const ll_recovery_cfg& c = R.cfg;
  cudaStream_t s = ctx->stream;
  // the map and its field, once per loss episode
  double t0 = now_ms();
  const ll_map* map = m->match_map;   // mode 0: the VoxelGrid of the live window, nothing appended since the first bad step
  if (!R.field_valid) {
    if (m->cfg.matching_mode == 1) {
      float4* vg[2]; int hc[2] = {0, 0};
      LL_TRY(whole_map_clouds(m, vg, hc));
      LL_TRY(ll_map_rebuild(ctx, R.whole, vg[0], (size_t)hc[0], vg[1], (size_t)hc[1], LL_FMT_XYZI16, LL_DEVICE));
    }
    if (m->cfg.matching_mode == 1) map = R.whole;
    LL_TRY(reloc_field_build_into(ctx, map, c.res, c.trunc, c.max_hypotheses, R.field));
    R.field_valid = true;
    e->ms_map = now_ms() - t0;
  }
  if (m->cfg.matching_mode == 1) map = R.whole;
  t0 = now_ms();
  // the step's features out of A.feat (the next step overwrites them) and the score points of each class
  RecoveryLayout rl; LL_CUDA(ctx, R.buf.carve([&](Carve& k) { rl.layout(k, (size_t)ctx->cfg.max_features); }));
  if (nc + ns > 0) LL_CUDA(ctx, cudaMemcpyAsync(rl.feat, ctx->A.feat, (size_t)(nc + ns) * 16, cudaMemcpyDeviceToDevice, s));
  int n_sc = 0, n_ss = 0;
  LL_TRY(score_points(ctx, rl.feat, nc, c.score_leaf, rl.score[0], rl.cnt, &n_sc, &e->score_leaf[0]));
  LL_TRY(score_points(ctx, rl.feat + nc, ns, c.score_leaf, rl.score[1], rl.cnt + 1, &n_ss, &e->score_leaf[1]));
  e->n_score[0] = n_sc; e->n_score[1] = n_ss;
  // coarse: the yaw circle x the tilt of the mapper's pose; the x / y lattice around its translation, clipped to the grid and max_hypotheses
  const double* q = m->q_w_curr; const double* t = m->t_w_curr;
  const double yaw = atan2(2.0 * (q[0] * q[3] + q[1] * q[2]), 1.0 - 2.0 * (q[2] * q[2] + q[3] * q[3]));
  double qy[4], qyc[4], tilt[4];
  yaw_quat(yaw * (180.0 / M_PI), qy);
  qyc[0] = qy[0]; qyc[1] = -qy[1]; qyc[2] = -qy[2]; qyc[3] = -qy[3];
  quat_mul(qyc, q, tilt);
  { const double nn = sqrt(tilt[0] * tilt[0] + tilt[1] * tilt[1] + tilt[2] * tilt[2] + tilt[3] * tilt[3]); for (int k = 0; k < 4; k++) tilt[k] /= nn; }
  const int n_yaw = coarse_yaws(c);
  R.rot_c.resize((size_t)n_yaw * 4);
  for (int k = 0; k < n_yaw; k++) { double a[4]; yaw_quat(k * (360.0 / n_yaw), a); quat_mul(a, tilt, &R.rot_c[(size_t)k * 4]); }
  int dims[3]; float lo[3];
  LL_TRY(ll_reloc_field_read(R.field, 0, dims, lo, nullptr, 0));
  const double W = c.window_base + c.window_growth * R.bad;
  const int h = (int)std::floor(W / c.t_step + 1e-9);
  int i0[2], i1[2];
  for (int a = 0; a < 2; a++) {
    const double glo = (double)lo[a], ghi = (double)lo[a] + (double)(dims[a] - 2 * c.trunc) * (double)c.res;
    i0[a] = std::max(-h, (int)std::ceil((glo - t[a]) / c.t_step));
    i1[a] = std::min(h, (int)std::floor((ghi - t[a]) / c.t_step));
    if (i0[a] > i1[a]) { i0[a] = i1[a] = 0; }   // the pose off the grid on this axis: its own coordinate only
  }
  const long long max_lat = c.max_hypotheses / n_yaw;
  while ((long long)(i1[0] - i0[0] + 1) * (i1[1] - i0[1] + 1) > max_lat) {   // shrink the wider axis at its end farther from the pose
    const int a = (i1[0] - i0[0]) >= (i1[1] - i0[1]) ? 0 : 1;
    if (-i0[a] > i1[a]) i0[a]++; else i1[a]--;
  }
  ll_reloc_cfg& co = R.coarse;
  memset(&co, 0, sizeof(co));
  co.n_rot = n_yaw; co.rot_wxyz = R.rot_c.data(); co.rot_cyclic = 1; co.max_candidates = c.max_candidates;
  for (int a = 0; a < 2; a++) { co.t0[a] = t[a] + i0[a] * c.t_step; co.step[a] = c.t_step; co.nt[a] = i1[a] - i0[a] + 1; }
  co.t0[2] = t[2]; co.step[2] = c.t_step; co.nt[2] = 1;
  // fine: the Python defaults (fine_search): yaw offsets +-yaw_step / 2, x / y +-fine_t_half coarse steps, one height
  const int nfy = fine_yaws(c), ny = nfy / 2;
  R.rot_f.resize((size_t)nfy * 4);
  for (int k = -ny; k <= ny; k++) yaw_quat(k * c.fine_yaw_step_deg, &R.rot_f[(size_t)(k + ny) * 4]);
  ll_reloc_fine_cfg& fi = R.fine;
  memset(&fi, 0, sizeof(fi));
  fi.n_rot = nfy; fi.rot_wxyz = R.rot_f.data();
  for (int a = 0; a < 3; a++) { fi.step[a] = c.fine_t_step; fi.nt[a] = a < 2 && co.nt[a] > 1 ? fine_nt(c) : 1; }
  R.tmpl = st;
  for (int a = 0; a < 3; a++) { e->t0[a] = co.t0[a]; e->step[a] = co.step[a]; e->nt[a] = co.nt[a]; }
  e->n_yaw = n_yaw;
  for (int k = 0; k < 4; k++) e->tilt_wxyz[k] = tilt[k];
  // K items of the step's features must fit max_features
  const int M = nc + ns;
  if (M > 0 && co.max_candidates * M > ctx->cfg.max_features) co.max_candidates = std::max(1, ctx->cfg.max_features / M);
  R.n_last[0] = (size_t)nc; R.n_last[1] = (size_t)ns; R.n_last[2] = (size_t)n_sc; R.n_last[3] = (size_t)n_ss;
  R.have_last = true;
  ll_reloc_field_candidate cand[LL_MAX_BATCH]; ll_reg_result refined[LL_MAX_BATCH]; int item_status[LL_MAX_BATCH]; int n_cand = 0, best = -1;
  const int rs = ll_relocalize_field(ctx, map, R.field, rl.score[0], (size_t)n_sc, rl.score[1], (size_t)n_ss, rl.feat, (size_t)nc, rl.feat + nc, (size_t)ns,
                                     LL_FMT_XYZI16, LL_DEVICE, &co, &fi, &R.tmpl, cand, refined, item_status, &n_cand, &best);
  e->ms_search = now_ms() - t0;
  LL_TRY(rs);
  e->n_cand = n_cand; e->best = best;
  if (best < 0) return LL_OK;
  const ll_reg_result& r = refined[best];
  const double T2 = (double)c.trunc * c.trunc;
  e->verify_fraction = n_sc + n_ss > 0 ? cand[best].verify_score / (T2 * (n_sc + n_ss)) : 0.0;
  for (int k = 0; k < 4; k++) e->q_wxyz[k] = r.q_w_curr[k];
  for (int k = 0; k < 3; k++) e->t[k] = r.t_w_curr[k];
  e->inlier_threshold = r.inlier_threshold;
  if (e->verify_fraction >= c.min_verify_fraction && r.inlier_threshold <= c.max_inlier_threshold) {
    mapper_set_pose(m, r.q_w_curr, r.t_w_curr);
    e->adopted = 1;
  }
  return LL_OK;
}

// The judgement of one registered step and, when the mapper is lost and the step is bad, an attempt.  *hold: the step is not appended.
static int recovery_step(ll_mapper* m, int nc, int ns, const ll_reg_state& st, const ll_reg_result* out, bool* hold) {
  Recovery& R = m->rec;
  const ll_recovery_cfg& c = R.cfg;
  ll_recovery_step* e = R.cur = R.log.push();
  e->frame_index = st.current_frame_index; e->state_before = R.state; e->best = -1;
  for (int k = 0; k < 4; k++) e->q_wxyz[k] = m->q_w_curr[k];
  for (int k = 0; k < 3; k++) e->t[k] = m->t_w_curr[k];
  if (out->registered == 1) {   // (a step that did not register, before the map exists or under :199, is not judged)
    if (out->status == 0) e->bad = LL_BAD_REJECTED;
    else if (!(out->inlier_threshold <= c.max_inlier_threshold)) e->bad = LL_BAD_INLIER;
    if (e->bad == LL_BAD_NONE) { R.bad = 0; R.state = LL_TRACKING; R.field_valid = false; }
    else {
      *hold = true;
      R.bad++;
      R.state = R.state == LL_LOST || R.bad >= c.lost_after ? LL_LOST : LL_SUSPECT;
      if (R.state == LL_LOST) {
        e->attempted = 1;
        const size_t b0 = buf_caps(m);
        const int as = recovery_attempt(m, nc, ns, st, e);
        e->grew = buf_caps(m) != b0 ? 1 : 0;
        e->attempt_status = as;
        if (as == LL_ERR_CUDA) return as;
      }
    }
  }
  e->bad_steps = R.bad; e->state_after = R.state;
  return LL_OK;
}

extern "C" {

void ll_mapper_recovery_default(ll_recovery_cfg* c) {
  if (!c) return;
  memset(c, 0, sizeof(*c));
  c->max_inlier_threshold = 0.1; c->lost_after = 3;           // DESIGN.md §4.3.2: normal C3-style scans stay below 0.045, kidnapped ones above 0.18
  c->res = 0.2f; c->trunc = 2; c->score_leaf = 0.5f;          // the field defaults of §4.3.1
  c->yaw_step_deg = 10.0; c->t_step = 1.0; c->window_base = 2.0; c->window_growth = 1.0; c->max_candidates = 8;
  c->fine_yaw_step_deg = 1.0; c->fine_t_step = 0.1; c->fine_t_half = 1.5;
  c->min_verify_fraction = 0.3;                               // the truth of a covered view scores 0.46 ... 0.76 (§4.3.2)
  c->max_hypotheses = 1 << 18;
  c->reserve_field_voxels = 1 << 22; c->reserve_whole_map_points = 1 << 20;
}

int ll_mapper_set_recovery(ll_mapper* m, const ll_recovery_cfg* cfg) {
  if (!m) return LL_ERR_INVALID;
  ll_ctx* ctx = m->ctx;
  Recovery& R = m->rec;
  if (!cfg) {
    R.on = false; R.state = LL_TRACKING; R.bad = 0; R.field_valid = false; R.have_last = false;
    ll_reloc_field_release(R.field); R.field = nullptr;
    if (R.whole) ll_map_release(R.whole);
    R.whole = nullptr; R.buf.release();
    return LL_OK;
  }
  if (const char* err = recovery_cfg_error(*cfg)) { ctx->set_error(std::string("recovery config: ") + err); return LL_ERR_INVALID; }
  cudaSetDevice(ctx->device);
  if (!R.field) R.field = reloc_field_create(ctx->device);
  if (!R.whole) { R.whole = new ll_map(); R.whole->device = ctx->device; }
  LL_TRY(reloc_field_reserve(ctx, R.field, cfg->reserve_field_voxels, cfg->max_hypotheses));
  RecoveryLayout rl; LL_CUDA(ctx, R.buf.reserve_floor(layout_bytes([&](Carve& k) { rl.layout(k, (size_t)ctx->cfg.max_features); })));
  if (m->cfg.matching_mode == 1 && cfg->reserve_whole_map_points > 0) {   // whole_map_clouds' feat_buf, VoxelGrid and index build
    const int W = (int)cfg->reserve_whole_map_points;
    LL_CUDA(ctx, ctx->feat_buf.reserve_floor((size_t)W * 4 * 16 + 64));
    const size_t side = std::max(voxel_grid_bytes(W), tree_scratch_bytes(W));
    LL_CUDA(ctx, ctx->scratch.reserve_floor(side)); LL_CUDA(ctx, ctx->scratch2.reserve_floor(side));
    for (BucketTree& t : R.whole->tree) LL_CUDA(ctx, t.storage.reserve_floor(tree_storage_bytes(W)));
  }
  R.log.open(LL_RECOVERY_LOG);
  R.cfg = *cfg; R.on = true; R.state = LL_TRACKING; R.bad = 0; R.field_valid = false;
  return LL_OK;
}

int ll_mapper_recovery_read(ll_mapper* m, ll_recovery_step* out, int cap, int* n, int* n_dropped) {
  if (!m || !n || cap < 0 || (cap > 0 && !out)) return LL_ERR_INVALID;
  m->rec.log.read(out, cap, n, n_dropped);
  return LL_OK;
}

int ll_mapper_recovery_last_inputs(ll_mapper* m, ll_reloc_cfg* coarse, ll_reloc_fine_cfg* fine, ll_reg_state* tmpl, size_t n[4], ll_point* corner, ll_point* surf,
                                   ll_point* score_corner, ll_point* score_surf, size_t cap_points, double* rot_coarse, double* rot_fine, int cap_rot) {
  if (!m || !n) return LL_ERR_INVALID;
  ll_ctx* ctx = m->ctx;
  Recovery& R = m->rec;
  if (!R.have_last) { ctx->set_error("no relocalization attempt yet"); return LL_ERR_INVALID; }
  for (int k = 0; k < 4; k++) n[k] = R.n_last[k];
  const int nrc = R.coarse.n_rot, nrf = R.fine.n_rot;
  ll_point* dst[4] = {corner, surf, score_corner, score_surf};
  for (int k = 0; k < 4; k++) if (dst[k] && cap_points < R.n_last[k]) return LL_ERR_CAPACITY;
  if ((rot_coarse && cap_rot < nrc) || (rot_fine && cap_rot < nrf)) return LL_ERR_CAPACITY;
  if (coarse) { *coarse = R.coarse; coarse->rot_wxyz = rot_coarse; }
  if (fine) { *fine = R.fine; fine->rot_wxyz = rot_fine; }
  if (tmpl) *tmpl = R.tmpl;
  if (rot_coarse) memcpy(rot_coarse, R.rot_c.data(), (size_t)nrc * 4 * sizeof(double));
  if (rot_fine) memcpy(rot_fine, R.rot_f.data(), (size_t)nrf * 4 * sizeof(double));
  cudaSetDevice(ctx->device);
  RecoveryLayout rl; LL_CUDA(ctx, R.buf.carve([&](Carve& k) { rl.layout(k, (size_t)ctx->cfg.max_features); }));   // (reserved: no reallocation)
  const float4* src[4] = {rl.feat, rl.feat + R.n_last[0], rl.score[0], rl.score[1]};
  for (int k = 0; k < 4; k++)
    if (dst[k] && R.n_last[k]) LL_CUDA(ctx, cudaMemcpyAsync(dst[k], src[k], R.n_last[k] * 16, cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return LL_OK;
}

// ---------------------------------------------------------------------------------------------- loop closure (loop.cu; DESIGN.md §4.6)
void ll_mapper_loop_closure_default(ll_loop_closure_cfg* c) {
  if (!c) return;
  memset(c, 0, sizeof(*c));
  c->scans_of_each_keyframe = 300; c->scans_between_two_keyframe = 100;            // performance_precision.yaml loop_closure/
  ll_loop_cfg_default(&c->loop); c->loop.minimum_keyframe_differen = 200;          // rosbag_loop.launch
  c->map_alignment_resolution = 0.1f; c->map_alignment_maximum_icp_iteration = 5; c->map_alignment_inlier_threshold = 0.20f;
  c->scene_alignment_maximum_residual_block = 3000;
  c->surround_pointcloud_resolution = 0.30;                                        // mapping/surround_pointcloud_resolution
  c->incremental_cov = 1;                                                          // common/if_update_mean_and_cov_incrementally
  c->rng_seed = 0; c->max_cells = 0;
  c->reserve_map_points = 1 << 22; c->reserve_history_points = 1 << 22; c->reserve_keyframes = 1024;
}

int ll_mapper_set_loop_closure(ll_mapper* m, const ll_loop_closure_cfg* cfg) {
  if (!m) return LL_ERR_INVALID;
  return loop_set(m->ctx, &m->lc, cfg, m->cfg, m->frame_pieces);
}

int ll_mapper_loop_read(ll_mapper* m, ll_loop_event* out, int cap, int* n, int* n_dropped) {
  if (!m || !n || cap < 0 || (cap > 0 && !out)) return LL_ERR_INVALID;
  return loop_read(m->lc, out, cap, n, n_dropped);
}

int ll_mapper_loop_result(ll_mapper* m, int* n, int* closed, ll_pose* poses_ori, ll_pose* poses_opt, int cap, ll_pg_edge* edge) {
  if (!m || cap < 0) return LL_ERR_INVALID;
  return loop_result(m->lc, n, closed, poses_ori, poses_opt, cap, edge);
}

int ll_mapper_loop_cloud(ll_mapper* m, int k, ll_point* out_host, size_t cap, size_t* n_out, const ll_point** out_dev) {
  if (!m || !n_out) return LL_ERR_INVALID;
  return loop_cloud(m->ctx, m->lc, k, out_host, cap, n_out, out_dev);
}

void ll_mapper_loop_policy_default(ll_loop_policy* p) {
  if (p) { p->max_loops = 1; p->min_keyframes_between_loops = 0; }
}

int ll_mapper_set_loop_policy(ll_mapper* m, const ll_loop_policy* p) {
  if (!m) return LL_ERR_INVALID;
  return loop_set_policy(m->ctx, m->lc, p);
}

int ll_mapper_loop_edges(ll_mapper* m, ll_pg_edge* edges, int cap, int* n_loops) {
  if (!m || !n_loops || cap < 0) return LL_ERR_INVALID;
  return loop_edges(m->lc, edges, cap, n_loops);
}

// The loop image's binding stamp: what the loop closure's state refers to in the mapper (loop.cu checks it on load).
static ll_loop_image_scalars loop_stamp(const ll_mapper* m) {
  ll_loop_image_scalars s; memset(&s, 0, sizeof(s));
  s.frame_index = m->frame_index; s.matching_mode = m->cfg.matching_mode; s.threshold_cell_revisit = m->cfg.threshold_cell_revisit;
  s.maximum_history_size = m->cfg.maximum_history_size; s.pieces = m->frame_pieces; s.cell_resolution = m->cfg.cell_resolution;
  s.last_time_stamp = m->last_time_stamp;
  for (int k = 0; k < 4; k++) s.q_w_curr[k] = m->q_w_curr[k];
  for (int k = 0; k < 3; k++) s.t_w_curr[k] = m->t_w_curr[k];
  return s;
}

int ll_mapper_loop_save(ll_mapper* m, void* image, size_t cap, size_t* bytes) {
  if (!m || !bytes) return LL_ERR_INVALID;
  if (!m->lc) { m->ctx->set_error("loop closure is off: there is no loop image"); return LL_ERR_INVALID; }
  cudaSetDevice(m->ctx->device);
  return loop_save(m->ctx, m->lc, loop_stamp(m), mapper_window(m), image, cap, bytes);
}

int ll_mapper_loop_load(ll_mapper* m, const void* image, size_t bytes, const ll_loop_closure_cfg* cfg) {
  if (!m) return LL_ERR_INVALID;
  return loop_load(m->ctx, &m->lc, image, bytes, cfg, loop_stamp(m), m->cfg, m->frame_pieces, mapper_window(m));
}

int ll_mapper_set_loop_feedback(ll_mapper* m, int on) {
  if (!m) return LL_ERR_INVALID;
  return loop_set_feedback(m->ctx, m->lc, m->cfg, on);
}

int ll_mapper_loop_correction_read(ll_mapper* m, double q_wxyz[4], double t[3], int* n_applied) {
  if (!m || !q_wxyz || !t) return LL_ERR_INVALID;
  loop_correction(m->lc, q_wxyz, t, n_applied);
  return LL_OK;
}

int ll_loop_image_info(const void* image, size_t bytes, ll_loop_image_summary* info) {
  if (!info) return LL_ERR_INVALID;
  return loop_image_info(image, bytes, info);
}

}  // extern "C"
