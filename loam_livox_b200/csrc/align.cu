// Loop-closure reuse of the registration hot path (SURVEY.md 8(f) N4): Scene_alignment::find_tranfrom_of_two_mappings
// (loam_livox/source/scene_alignment.hpp:269-353, object set-up :233-243): the same find_out_incremental_transfrom, called three times,
// coarse to fine (leaf x8, x4, x1), with ICP_LINE = 0, on ONE persistent Point_cloud_registration object -- so m_para_buffer_incremental
// (q_incre, t_incre), m_q_w_curr and m_t_w_curr carry over from one scale to the next while m_q_w_last / m_t_w_last stay (identity, 0).
// The four feature clouds (line / plane points of the two keyframes) are the caller's; extracting them (cell eigen-analysis, Maps_keyframe)
// is outside the hot path.  Everything below is host orchestration of entry points that already exist: VoxelGrid, index build, registration.
#include <cmath>
#include <cstring>
#include "common.cuh"
#include "kernels.cuh"

extern "C" {

void ll_align_cfg_default(ll_align_cfg* c) {
  memset(c, 0, sizeof(*c));
  c->line_res = 0.4f; c->plane_res = 0.4f;          // scene_alignment.hpp:27-28
  c->maximum_icp_iteration = 10;                    // :35
  c->maximum_residual_block = 5000;                 // :34
  c->accepted_threshold = 0.2f;                     // :36
  c->rng_seed = 0;
}

int ll_scene_align(ll_ctx* ctx, const void* src_line, size_t n_sl, const void* src_plane, size_t n_sp, const void* tgt_line, size_t n_tl, const void* tgt_plane, size_t n_tp,
                   int fmt, int where, const ll_align_cfg* cfg, ll_reg_result* out, int* scales_run) {
  if (!ctx || !cfg || !out) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  cudaStream_t s = ctx->stream;
  const size_t ns[4] = {n_sl, n_sp, n_tl, n_tp}; const void* srcs[4] = {src_line, src_plane, tgt_line, tgt_plane};
  if ((int)(n_tl + n_tp) > ctx->cfg.max_features) { ctx->set_error("more target features than max_features"); return LL_ERR_CAPACITY; }
  // the four input clouds and their down-sampled versions, on the device (one arena)
  float4* d_in[4]; float4* d_ds[4]; int* d_cnt;
  DevBuf arena;   // released on every exit path below
  LL_CUDA(ctx, arena.carve([&](Carve& c) {
    for (int k = 0; k < 4; k++) d_in[k] = c.take<float4>(ns[k] + 1);
    for (int k = 0; k < 4; k++) d_ds[k] = c.take<float4>(ns[k] + 1);
    d_cnt = c.take<int>(4);
  }));
  auto fail = [&](int st) { arena.release(); return st; };
  for (int k = 0; k < 4; k++) { const int st = upload_cloud(ctx, srcs[k], ns[k], fmt, where, d_in[k]); if (st != LL_OK) return fail(st); }
  // m_pc_reg as set_up_log_dir / find_tranfrom_of_two_mappings leave it (:233-243, :292-306)
  ll_reg_state st; ll_reg_state_default(&st);
  st.icp_line = 0; st.icp_plane = 1;
  st.max_final_cost = 20000; st.para_max_speed = 1000.0; st.para_max_angular_rate = 360 * 57.3; st.inliner_dis = 0.2;
  st.current_frame_index = 10000000; st.mapping_init_accumulate_frames = 100;
  st.icp_max_iterations = cfg->maximum_icp_iteration; st.cere_max_iterations = 50; st.cere_prerun_times = 2;
  st.maximum_allow_residual_block = cfg->maximum_residual_block; st.rng_seed = cfg->rng_seed;
  st.q_w_last[0] = 1; st.q_w_last[1] = st.q_w_last[2] = st.q_w_last[3] = 0; st.t_w_last[0] = st.t_w_last[1] = st.t_w_last[2] = 0;
  st.q_w_curr[0] = 1; st.q_w_curr[1] = st.q_w_curr[2] = st.q_w_curr[3] = 0;
  for (int k = 0; k < 3; k++) { st.t_w_curr[k] = cfg->t_init[k]; st.para_buffer_incremental[4 + k] = cfg->t_init[k]; }   // m_t_w_incre = m_t_w_curr = transform_T
  st.para_buffer_incremental[0] = st.para_buffer_incremental[1] = st.para_buffer_incremental[2] = 0; st.para_buffer_incremental[3] = 1;
  memset(out, 0, sizeof(*out)); out->status = 1;
  for (int k = 0; k < 4; k++) out->q_w_curr[k] = st.q_w_curr[k]; for (int k = 0; k < 3; k++) out->t_w_curr[k] = st.t_w_curr[k];
  int runs = 0;
  ll_map* map = nullptr;
  for (int scale = 8; scale >= 0; scale -= 4) {
    float line_res = cfg->line_res * scale, plane_res = cfg->plane_res * scale;
    if (line_res < cfg->line_res) line_res = cfg->line_res;
    if (plane_res < cfg->plane_res) { plane_res = cfg->plane_res; st.icp_max_iterations = cfg->maximum_icp_iteration * 2; }
    const float leaf[4] = {line_res, plane_res, line_res, plane_res};
    int h_cnt[4] = {0, 0, 0, 0};
    for (int k = 0; k < 4; k++) {
      if (ns[k] == 0) { cudaMemsetAsync(d_cnt + k, 0, 4, s); continue; }
      const int stv = launch_voxel_grid(ctx, s, ctx->scratch, d_in[k], (int)ns[k], nullptr, leaf[k], d_ds[k], d_cnt + k);
      if (stv != LL_OK) { if (map) ll_map_release(map); return fail(stv); }
    }
    if (cudaMemcpyAsync(h_cnt, d_cnt, sizeof(h_cnt), cudaMemcpyDeviceToHost, s) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess) { if (map) ll_map_release(map); return fail(LL_ERR_CUDA); }
    runs++;
    if (h_cnt[0] == 0 || h_cnt[1] == 0) continue;   // the 4-argument overload returns 1 without touching anything (:595-603)
    int stm = map ? ll_map_rebuild(ctx, map, d_ds[0], (size_t)h_cnt[0], d_ds[1], (size_t)h_cnt[1], LL_FMT_XYZI16, LL_DEVICE)
                  : ll_map_build(ctx, d_ds[0], (size_t)h_cnt[0], d_ds[1], (size_t)h_cnt[1], LL_FMT_XYZI16, LL_DEVICE, &map);
    if (stm != LL_OK) { if (map) ll_map_release(map); return fail(stm); }
    ll_reg_result r;
    const int str = ll_register(ctx, map, d_ds[2], (size_t)h_cnt[2], d_ds[3], (size_t)h_cnt[3], LL_FMT_XYZI16, LL_DEVICE, &st, &r);
    if (str != LL_OK) { ll_map_release(map); return fail(str); }
    *out = r;
    // the object persists: pose and increment carry over to the next scale; q_w_last / t_w_last stay (identity, 0)
    for (int k = 0; k < 4; k++) st.q_w_curr[k] = r.q_w_curr[k]; for (int k = 0; k < 3; k++) st.t_w_curr[k] = r.t_w_curr[k];
    st.para_buffer_incremental[0] = r.q_w_incre[1]; st.para_buffer_incremental[1] = r.q_w_incre[2]; st.para_buffer_incremental[2] = r.q_w_incre[3]; st.para_buffer_incremental[3] = r.q_w_incre[0];
    for (int k = 0; k < 3; k++) st.para_buffer_incremental[4 + k] = r.t_w_incre[k];
    if (r.registered && r.inlier_threshold > (double)(cfg->accepted_threshold * 2)) break;   // :349-350
  }
  if (scales_run) *scales_run = runs;
  if (map) ll_map_release(map);
  arena.release();
  return LL_OK;
}

}  // extern "C"
