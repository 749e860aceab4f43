// C-ABI of libloamlivox_b200.so (see include/loamlivox_b200.h) and the host-side ICP driver.
//
// Host logic restated from Point_cloud_registration::find_out_incremental_transfrom
// (loam_livox/source/point_cloud_registration.hpp:163-583): the gate at :199, the ICP loop :211-532 (the per-iteration work is
// four kernels: kNN+blocks, solve #1, inlier select, solve #2 + pose/termination), the threshold rescale :559 and the reject gate :561-573.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <cstdlib>
#include <cstdio>
#include "common.cuh"
#include "kernels.cuh"

// Everything whose size the config fixes, laid out once at creation: the registration arrays (max_features slots; the front end's feature
// clouds: max_scan_points), the extractor's arrays and the front end's scratch arenas.  Callers reject more than max_features slots, so none of
// this moves afterwards.
static int ctx_alloc(ll_ctx* ctx) {
  const size_t cap = (size_t)ctx->cfg.max_features, scap = ctx->cfg.max_scan_points > ctx->cfg.max_features ? (size_t)ctx->cfg.max_scan_points : cap;
  RegArrays& A = ctx->A;
  LL_CUDA(ctx, ctx->reg_buf.carve([&](Carve& c) {
    A.feat = c.take<float4>(cap); A.blk_a = c.take<float4>(cap); A.blk_v = c.take<double>(cap * 3);
    A.l1 = c.take<double>(cap); A.k10_value = c.take<double>(1);
    A.k10_n_distinct = c.take<int>(1); A.counts = c.take<int>(16); A.bounds = c.take<float>(32);
    A.knn_idx = c.take<int>(cap * LL_KNN); A.knn_d = c.take<float>(cap * LL_KNN); A.perm = c.take<int>(cap);
    A.tmp_a = c.take<float4>(scap); A.tmp_b = c.take<float4>(scap); A.tmp_c = c.take<float4>(scap); A.tmp_d = c.take<float4>(scap);
    A.dev_counts = c.take<int>(2);
  }));
  LL_TRY(extract_alloc(ctx));
  // the front end: extraction + get_features + the surface VoxelGrids on fe_main, the corner VoxelGrids on fe_corner, the petals on fe_petals
  const int n = ctx->cfg.max_scan_points;
  const size_t vg = voxel_grid_bytes(n), pet = petals_bytes(n), gf = get_features_bytes(n);
  LL_CUDA(ctx, ctx->fe_main.reserve(std::max(vg, std::max(pet, gf))));
  LL_CUDA(ctx, ctx->fe_corner.reserve(vg));
  LL_CUDA(ctx, ctx->fe_petals.reserve(pet));
  return LL_OK;
}

extern "C" {

void ll_config_default(ll_config* c) {
  c->corner_curvature = 0.1f; c->surface_curvature = 0.005f; c->minimum_view_angle = 5.0f; c->livox_min_dis = 0.1f; c->livox_min_sigma = 7e-4f;
  c->max_fov_deg = 17.0f; c->time_interval_pts = 1.0e-5f; c->max_scan_points = 400000; c->max_features = 400000;
}
void ll_reg_state_default(ll_reg_state* s) {
  memset(s, 0, sizeof(*s));
  s->if_motion_deblur = 0; s->current_frame_index = 1000; s->mapping_init_accumulate_frames = 50; s->icp_max_iterations = 15; s->cere_max_iterations = 50; s->cere_prerun_times = 2;
  s->icp_plane = 1; s->icp_line = 1; s->maximum_allow_residual_block = 1000000;
  s->para_max_angular_rate = 20.0; s->para_max_speed = 0.3; s->max_final_cost = 1.0e9; s->minimum_pt_time_stamp = 0.0; s->maximum_pt_time_stamp = 0.1;
  s->minimum_icp_R_diff = 0.01; s->minimum_icp_T_diff = 0.01; s->inliner_dis = 0.02; s->inlier_ratio = 0.80; s->maximum_dis_plane_for_match = 50.0; s->maximum_dis_line_for_match = 2.0; s->huber_a = 0.1;
  s->q_w_last[0] = 1; s->q_w_curr[0] = 1; s->para_buffer_incremental[3] = 1;
}

void ll_reg_state_yaml(ll_reg_state* s, int realtime) {
  ll_reg_state_default(s);
  s->maximum_allow_residual_block = realtime ? 150 : 200;   // config/performance_realtime.yaml:23 / performance_precision.yaml:23
  s->max_final_cost = 2.0;                                  // optimization/max_allow_final_cost
}
float ll_cap_uniform(int seed, int icp_iteration, int stream, int index) { return ll_cap_uniform_f(seed, icp_iteration, stream, index); }

int ll_ctx_create(const ll_config* cfg, int device, ll_ctx** out) {
  if (!out) return LL_ERR_INVALID;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return LL_ERR_CUDA;   // no silent CPU fallback: the CUDA path is the product
  if (device < 0 || device >= ndev) return LL_ERR_INVALID;
  // ex_scatter_kernel packs the three running counts of get_features in 21 bits each; the cap on a scan is therefore 2^21 - 1 points
  if (cfg && (cfg->max_scan_points < 1 || cfg->max_scan_points >= (1 << 21) || cfg->max_features < 1)) return LL_ERR_INVALID;
  ll_ctx* ctx = new ll_ctx();
  ctx->device = device;
  if (cfg) ctx->cfg = *cfg; else ll_config_default(&ctx->cfg);
  // every call is checked: the first failure wins and the half-built context is torn down by ll_ctx_destroy (which tolerates null members)
  cudaError_t e = cudaSetDevice(device);
  auto ok = [&](cudaError_t r) { if (e == cudaSuccess && r != cudaSuccess) e = r; };
  cudaDeviceProp prop; ok(cudaGetDeviceProperties(&prop, device)); ctx->num_sms = prop.multiProcessorCount;
  // the context's own streams at the greatest priority, the sequence calls' front end at the least: the front end of the next input only takes
  // what the mapper step leaves of the GPU (every stream of the single-input calls has the same priority, so their scheduling is as before)
  int least = 0, greatest = 0; ok(cudaDeviceGetStreamPriorityRange(&least, &greatest));
  for (cudaStream_t* s : {&ctx->stream, &ctx->stream2, &ctx->stream3}) ok(cudaStreamCreateWithPriority(s, cudaStreamNonBlocking, greatest));
  for (cudaStream_t& s : ctx->fe_stream) ok(cudaStreamCreateWithPriority(&s, cudaStreamNonBlocking, least));
  ctx->sev.each([&](cudaEvent_t& ev) { ok(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)); });
  ctx->ev.each([&](cudaEvent_t& ev) { ok(cudaEventCreate(&ev)); });
  ok(cudaHostAlloc((void**)&ctx->pin, sizeof(PinnedStage), cudaHostAllocDefault));
  // one registration state per batch item (d_reg[0]: ll_register and the parity hooks)
  void* dreg = nullptr; ok(cudaMalloc(&dreg, LL_MAX_BATCH * sizeof(RegDevState))); if (dreg) ok(cudaMemset(dreg, 0, LL_MAX_BATCH * sizeof(RegDevState))); ctx->d_reg = (RegDevState*)dreg;
  if (e == cudaSuccess && solve_prepare(ctx) != LL_OK) e = cudaErrorUnknown;   // per-function attributes of the solver kernels (no process-global flag: contexts are created from any thread)
  if (e == cudaSuccess && voxel_grid_prepare(ctx) != LL_OK) e = cudaErrorUnknown;
  if (e == cudaSuccess && ctx_alloc(ctx) != LL_OK) e = cudaErrorMemoryAllocation;
  if (e != cudaSuccess) { cudaGetLastError(); ll_ctx_destroy(ctx); return LL_ERR_CUDA; }
  *out = ctx; return LL_OK;
}
void ll_ctx_destroy(ll_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  for (cudaStream_t s : {ctx->stream, ctx->stream2, ctx->stream3, ctx->fe_stream[0], ctx->fe_stream[1], ctx->fe_stream[2]}) if (s) cudaStreamSynchronize(s);
  if (ctx->fg.exec) cudaGraphExecDestroy(ctx->fg.exec);
  for (DevBuf* b : {&ctx->scratch, &ctx->scratch2, &ctx->fe_main, &ctx->fe_corner, &ctx->fe_petals, &ctx->stage_in, &ctx->extract_buf, &ctx->feat_buf, &ctx->reg_buf}) b->release();
  if (ctx->pin) cudaFreeHost(ctx->pin);
  if (ctx->d_reg) cudaFree(ctx->d_reg);
  if (ctx->d_sync) cudaFree(ctx->d_sync);
  if (ctx->comm_local) cudaFree(ctx->comm_local);
  for (int i = 0; i < 8; i++) if (ctx->comm_peers[i] && i != ctx->rank) cudaIpcCloseMemHandle(ctx->comm_peers[i]);
  ctx->sev.each([](cudaEvent_t& ev) { if (ev) cudaEventDestroy(ev); });
  ctx->ev.each([](cudaEvent_t& ev) { if (ev) cudaEventDestroy(ev); });
  for (cudaStream_t s : {ctx->fe_stream[2], ctx->fe_stream[1], ctx->fe_stream[0], ctx->stream3, ctx->stream2, ctx->stream}) if (s) cudaStreamDestroy(s);
  delete ctx;
}
const char* ll_last_error(const ll_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }
void* ll_ctx_stream(ll_ctx* ctx) { return (void*)ctx->stream; }
int ll_ctx_sync(ll_ctx* ctx) { cudaSetDevice(ctx->device); LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); return LL_OK; }
uint64_t ll_launch_count(const ll_ctx* ctx) { return ctx->launches; }

// ---------------------------------------------------------------------------------------------- S1
// Host half of extract_laser_features: time-stamp bookkeeping (:724-736), upload, scan time to the device (staged through `pin_time`, by
// default the single extract_time slot), on stream s.
// The time-stamp bookkeeping alone (host): returns m_current_time of a scan of n points stamped `stamp`.
static double extract_stamp(ll_ctx* ctx, size_t n, double stamp) {
  ExtractState& e = ctx->ex;
  if (stamp <= 0.0000001 || (stamp < e.last_maximum_time_stamp)) e.current_time = e.last_maximum_time_stamp; else e.current_time = stamp - e.first_receive_time;
  if (e.first_receive_time <= 0) e.first_receive_time = stamp;
  e.n = (int)n;
  if (n > 0) e.last_maximum_time_stamp = (double)(float)(e.current_time + (double)(((float)(n - 1)) * ctx->cfg.time_interval_pts));
  return e.current_time;
}
static int extract_prepare(ll_ctx* ctx, cudaStream_t s, const void* raw, size_t n, int fmt, int where, double stamp, double* pin_time = nullptr) {
  if ((int)n > ctx->cfg.max_scan_points) { ctx->set_error("scan larger than max_scan_points"); return LL_ERR_CAPACITY; }
  ExtractState& e = ctx->ex;
  extract_stamp(ctx, n, stamp);
  LL_TRY(upload_cloud(ctx, s, raw, n, fmt, where, e.raw));
  if (!pin_time) pin_time = &ctx->pin->extract_time;
  *pin_time = e.current_time;
  LL_CUDA(ctx, cudaMemcpyAsync(e.d_time, pin_time, sizeof(double), cudaMemcpyHostToDevice, s));
  return LL_OK;
}
// The extraction on stream s; the petal bookkeeping's temporaries in `scratch`.
static int extract_enqueue(ll_ctx* ctx, cudaStream_t s, DevBuf& scratch) {
  ExtractState& e = ctx->ex;
  if (e.n > 0) { LL_TRY(launch_extract_points(ctx, s, e.n)); LL_TRY(launch_extract_petals(ctx, e.n, s, scratch)); }   // every size: get_features reads the per-point state
  else LL_CUDA(ctx, cudaMemsetAsync(e.d_meta, 0, 16, s));
  return LL_OK;
}
int ll_extract(ll_ctx* ctx, const void* raw, size_t n, int fmt, int where, double stamp, int* n_scans) {
  if (!ctx || (!raw && n)) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  ExtractState& e = ctx->ex;
  LL_TRY(extract_prepare(ctx, ctx->stream, raw, n, fmt, where, stamp));
  LL_TRY(extract_enqueue(ctx, ctx->stream, ctx->scratch));
  if (n_scans) {
    int* h = ctx->pin->counts;
    LL_CUDA(ctx, cudaMemcpyAsync(h, e.d_meta, 3 * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *n_scans = h[1];
  }
  return LL_OK;
}
int ll_extract_reset(ll_ctx* ctx) {
  if (!ctx) return LL_ERR_INVALID;
  ctx->ex.first_receive_time = -1; ctx->ex.current_time = 0; ctx->ex.last_maximum_time_stamp = 0; ctx->ex.n = 0;
  return LL_OK;
}
int ll_piece_bounds(ll_ctx* ctx, int pieces, float* start, float* end) {
  if (!ctx || pieces < 1 || pieces > 16) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  const RegArrays& A = ctx->A;
  LL_TRY(launch_piece_bounds(ctx, ctx->stream, pieces, A.bounds));
  float* h = ctx->pin->bounds;
  LL_CUDA(ctx, cudaMemcpyAsync(h, A.bounds, 2 * pieces * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < pieces; i++) { start[i] = h[2 * i]; end[i] = h[2 * i + 1]; }
  return LL_OK;
}
int ll_get_features(ll_ctx* ctx, float minimum_blur, float maximum_blur, ll_point* corners, size_t* n_corners, ll_point* surface, size_t* n_surface, ll_point* full, size_t* n_full) {
  if (!ctx) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  const RegArrays& A = ctx->A;
  LL_TRY(launch_get_features(ctx, ctx->stream, ctx->scratch, nullptr, minimum_blur, maximum_blur, A.tmp_a, A.tmp_b, A.tmp_c, A.counts));
  int* h = ctx->pin->counts;
  LL_CUDA(ctx, cudaMemcpyAsync(h, A.counts, 3 * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  int nc = ctx->ex.n ? h[0] : 0, ns = ctx->ex.n ? h[1] : 0, nf = ctx->ex.n ? h[2] : 0;
  if (corners && nc) LL_CUDA(ctx, cudaMemcpyAsync(corners, A.tmp_a, (size_t)nc * 16, cudaMemcpyDeviceToHost, ctx->stream));
  if (surface && ns) LL_CUDA(ctx, cudaMemcpyAsync(surface, A.tmp_b, (size_t)ns * 16, cudaMemcpyDeviceToHost, ctx->stream));
  if (full && nf) LL_CUDA(ctx, cudaMemcpyAsync(full, A.tmp_c, (size_t)nf * 16, cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (n_corners) *n_corners = nc; if (n_surface) *n_surface = ns; if (n_full) *n_full = nf;
  return LL_OK;
}
int ll_extract_point_info(ll_ctx* ctx, int32_t* pt_type, int32_t* pt_label, float* curvature, float* view_angle, float* depth_sq2, float* time_stamp, float* polar_dis_sq2, int32_t* polar_direction) {
  if (!ctx) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  ExtractState& e = ctx->ex; size_t n = e.n; cudaStream_t s = ctx->stream;
  if (pt_type) LL_CUDA(ctx, cudaMemcpyAsync(pt_type, e.pt_type, n * 4, cudaMemcpyDeviceToHost, s));
  if (pt_label) LL_CUDA(ctx, cudaMemcpyAsync(pt_label, e.pt_label, n * 4, cudaMemcpyDeviceToHost, s));
  if (curvature) LL_CUDA(ctx, cudaMemcpyAsync(curvature, e.curvature, n * 4, cudaMemcpyDeviceToHost, s));
  if (view_angle) LL_CUDA(ctx, cudaMemcpyAsync(view_angle, e.view_angle, n * 4, cudaMemcpyDeviceToHost, s));
  if (depth_sq2) LL_CUDA(ctx, cudaMemcpyAsync(depth_sq2, e.depth_sq2, n * 4, cudaMemcpyDeviceToHost, s));
  if (time_stamp) LL_CUDA(ctx, cudaMemcpyAsync(time_stamp, e.time_stamp, n * 4, cudaMemcpyDeviceToHost, s));
  if (polar_dis_sq2) LL_CUDA(ctx, cudaMemcpyAsync(polar_dis_sq2, e.polar_dis_sq2, n * 4, cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  if (polar_direction) {
    std::vector<int8_t> tmp(n);
    LL_CUDA(ctx, cudaMemcpy(tmp.data(), e.polar_dir, n, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < n; i++) polar_direction[i] = tmp[i];
  }
  return LL_OK;
}
int ll_extract_split_idx(ll_ctx* ctx, int32_t* out, int cap, int* n_out) {
  if (!ctx) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  int meta[3] = {0, 0, 0};
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  LL_CUDA(ctx, cudaMemcpy(meta, ctx->ex.d_meta, sizeof(meta), cudaMemcpyDeviceToHost));
  int m = meta[0] < cap ? meta[0] : cap;
  if (m > 0) LL_CUDA(ctx, cudaMemcpy(out, ctx->ex.split_idx, (size_t)m * 4, cudaMemcpyDeviceToHost));
  if (n_out) *n_out = meta[0];
  return LL_OK;
}
int ll_extract_petal_angles(ll_ctx* ctx, float* out, int cap, int* n_out) {
  if (!ctx) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  int meta[3] = {0, 0, 0};
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  LL_CUDA(ctx, cudaMemcpy(meta, ctx->ex.d_meta, sizeof(meta), cudaMemcpyDeviceToHost));
  const int nseg = meta[0] >= 6 ? meta[0] - 1 : 0;   // the angles exist only when the scan has enough split indices for petals
  const int m = nseg < cap ? nseg : cap;
  if (m > 0) LL_CUDA(ctx, cudaMemcpy(out, ctx->ex.seg_angle, (size_t)m * 4, cudaMemcpyDeviceToHost));
  if (n_out) *n_out = nseg;
  return LL_OK;
}

// ---------------------------------------------------------------------------------------------- a5 / a7
int ll_voxel_downsample(ll_ctx* ctx, const void* in, size_t n, int fmt, int where, float leaf, ll_point* out, size_t* n_out) {
  if (!ctx || !n_out || !(leaf > 0.f)) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  *n_out = 0; if (n == 0) return LL_OK;
  float4* d_in; float4* d_out; int* d_n;
  LL_CUDA(ctx, ctx->feat_buf.carve([&](Carve& c) { d_in = c.take<float4>(n); d_out = c.take<float4>(n); d_n = c.take<int>(1); }));
  LL_TRY(upload_cloud(ctx, ctx->stream, in, n, fmt, where, d_in));
  LL_TRY(launch_voxel_grid(ctx, ctx->stream, ctx->scratch, d_in, (int)n, nullptr, leaf, d_out, d_n));
  int* h = ctx->pin->counts;
  LL_CUDA(ctx, cudaMemcpyAsync(h, d_n, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  *n_out = (size_t)h[0];
  if (out && h[0] > 0) { LL_CUDA(ctx, cudaMemcpyAsync(out, d_out, (size_t)h[0] * 16, cudaMemcpyDeviceToHost, ctx->stream)); LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); }
  return LL_OK;
}
int ll_voxel_downsample_segments(ll_ctx* ctx, const ll_point* in, size_t n, const size_t* seg_end, int n_seg, float leaf, ll_point* out, size_t* n_out_per_seg) {
  if (!ctx || !seg_end || !n_out_per_seg || (!in && n) || n_seg < 1 || n_seg > 256 || !(leaf > 0.f) || n >= (size_t)1 << 31) return LL_ERR_INVALID;
  for (int k = 0; k < n_seg; k++) if (seg_end[k] > n || (k && seg_end[k] < seg_end[k - 1])) { ctx->set_error("segment ends must ascend and stay within n"); return LL_ERR_INVALID; }
  cudaSetDevice(ctx->device);
  cudaStream_t s = ctx->stream;
  float4* d_in = nullptr; float4* d_out = nullptr; int* d_end; int* d_oend;
  LL_CUDA(ctx, ctx->feat_buf.carve([&](Carve& c) { d_in = c.take<float4>(n); d_out = c.take<float4>(n); d_end = c.take<int>(n_seg); d_oend = c.take<int>(n_seg); }));
  std::vector<int> h(n_seg); for (int k = 0; k < n_seg; k++) h[k] = (int)seg_end[k];
  LL_CUDA(ctx, cudaMemcpyAsync(d_end, h.data(), n_seg * sizeof(int), cudaMemcpyHostToDevice, s));
  LL_TRY(upload_cloud(ctx, ctx->stream, in, n, LL_FMT_XYZI16, LL_HOST, d_in));
  LL_TRY(launch_voxel_grid_segments(ctx, s, ctx->scratch, d_in, (int)n, d_end, n_seg, leaf, d_out, d_oend));
  LL_CUDA(ctx, cudaMemcpyAsync(h.data(), d_oend, n_seg * sizeof(int), cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  for (int k = 0; k < n_seg; k++) n_out_per_seg[k] = (size_t)(h[k] - (k ? h[k - 1] : 0));
  if (out && h[n_seg - 1] > 0) { LL_CUDA(ctx, cudaMemcpyAsync(out, d_out, (size_t)h[n_seg - 1] * 16, cudaMemcpyDeviceToHost, s)); LL_CUDA(ctx, cudaStreamSynchronize(s)); }
  return LL_OK;
}
int ll_transform(ll_ctx* ctx, const double q[4], const double t[3], const void* in, size_t n, int fmt, int where, ll_point* out) {
  if (!ctx || !q || !t) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  if (n == 0) return LL_OK;
  float4* d_in; float4* d_out; double* d_pose;
  LL_CUDA(ctx, ctx->feat_buf.carve([&](Carve& c) { d_in = c.take<float4>(n); d_out = c.take<float4>(n); d_pose = c.take<double>(7); }));
  double* h = ctx->pin->pose; for (int k = 0; k < 4; k++) h[k] = q[k]; for (int k = 0; k < 3; k++) h[4 + k] = t[k];
  LL_CUDA(ctx, cudaMemcpyAsync(d_pose, h, 7 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  LL_TRY(upload_cloud(ctx, ctx->stream, in, n, fmt, where, d_in));
  LL_TRY(launch_transform(ctx, ctx->stream, d_pose, d_in, (int)n, d_out));
  LL_CUDA(ctx, cudaMemcpyAsync(out, d_out, n * 16, cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return LL_OK;
}

int ll_voxel_downsample_dev(ll_ctx* ctx, const ll_point* in_dev, size_t n, float leaf, ll_point* out_dev, size_t* n_out) {
  if (!ctx || !n_out || !(leaf > 0.f)) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  *n_out = 0; if (n == 0) return LL_OK;
  int* d_n;
  LL_CUDA(ctx, ctx->feat_buf.carve([&](Carve& c) { d_n = c.take<int>(1); }));
  LL_TRY(launch_voxel_grid(ctx, ctx->stream, ctx->scratch, (const float4*)in_dev, (int)n, nullptr, leaf, (float4*)out_dev, d_n));
  int* h = ctx->pin->counts;
  LL_CUDA(ctx, cudaMemcpyAsync(h, d_n, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  *n_out = (size_t)h[0];
  return LL_OK;
}
int ll_transform_dev(ll_ctx* ctx, const double q[4], const double t[3], const ll_point* in_dev, size_t n, ll_point* out_dev) {
  if (!ctx || !q || !t) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  if (n == 0) return LL_OK;
  double* d_pose;
  LL_CUDA(ctx, ctx->feat_buf.carve([&](Carve& c) { d_pose = c.take<double>(7); }));
  double* h = ctx->pin->pose; for (int k = 0; k < 4; k++) h[k] = q[k]; for (int k = 0; k < 3; k++) h[4 + k] = t[k];
  LL_CUDA(ctx, cudaMemcpyAsync(d_pose, h, 7 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  LL_TRY(launch_transform(ctx, ctx->stream, d_pose, (const float4*)in_dev, (int)n, (float4*)out_dev));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return LL_OK;
}
int ll_last_features_dev(ll_ctx* ctx, const ll_point** corner_dev, size_t* n_corner, const ll_point** surf_dev, size_t* n_surf) {
  if (!ctx) return LL_ERR_INVALID;
  const RegArrays& A = ctx->A;
  if (corner_dev) *corner_dev = (const ll_point*)A.feat; if (n_corner) *n_corner = (size_t)ctx->last_nc;
  if (surf_dev) *surf_dev = (const ll_point*)(A.feat + ctx->last_nc); if (n_surf) *n_surf = (size_t)ctx->last_ns;
  return LL_OK;
}

// ---------------------------------------------------------------------------------------------- S2
static int map_index(ll_ctx* ctx, ll_map* m, const void* corner, size_t nc, const void* surf, size_t ns, int fmt, int where) {
  // device clouds already in the library's layout are indexed where they lie (the tree keeps its own source-order copy)
  const bool in_place = where == LL_DEVICE && fmt == LL_FMT_XYZI16;
  const float4* d_c = (const float4*)corner; const float4* d_s = (const float4*)surf;
  int st = LL_OK;
  if (!in_place) {
    float4* b_c; float4* b_s;
    LL_CUDA(ctx, ctx->feat_buf.carve([&](Carve& c) { b_c = c.take<float4>(nc); b_s = c.take<float4>(ns); }));
    d_c = b_c; d_s = b_s;
    st = upload_cloud(ctx, ctx->stream, corner, nc, fmt, where, b_c);
    if (st == LL_OK) st = upload_cloud(ctx, ctx->stream, surf, ns, fmt, where, b_s);
    if (st != LL_OK) return st;
  }
  cudaStream_t s = ctx->stream;
  const float4* src[2] = {d_c, d_s}; const size_t n[2] = {nc, ns};
  st = map_side_pair(ctx, s, [&](int c, cudaStream_t cs, DevBuf& scr) { return build_bucket_tree(ctx, cs, scr, src[c], (int)n[c], &m->tree[c]); });
  // host inputs may be freed by the caller as soon as this returns; device inputs are consumed in stream order (the per-scan refresh never waits)
  if (st == LL_OK && where == LL_HOST && cudaStreamSynchronize(s) != cudaSuccess) st = LL_ERR_CUDA;
  return st;
}
static int map_build_common(ll_ctx* ctx, const void* corner, size_t nc, const void* surf, size_t ns, int fmt, int where, ll_map** out) {
  if (!ctx || !out) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  ll_map* m = new ll_map(); m->device = ctx->device;
  int st = map_index(ctx, m, corner, nc, surf, ns, fmt, where);
  if (st != LL_OK) { ll_map_release(m); return st; }
  *out = m; return LL_OK;
}
// Re-index an existing snapshot in place (device buffers are reused when large enough): the per-scan refresh of
// update_buff_for_matching (laser_mapping.hpp:544-545) without an allocation per scan.  The caller must not be searching `map` concurrently.
int ll_map_rebuild(ll_ctx* ctx, ll_map* map, const void* corner, size_t nc, const void* surf, size_t ns, int fmt, int where) {
  if (!ctx || !map) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  return map_index(ctx, map, corner, nc, surf, ns, fmt, where);
}
int ll_map_build(ll_ctx* ctx, const void* corner, size_t nc, const void* surf, size_t ns, int fmt, int where, ll_map** out) {
  return map_build_common(ctx, corner, nc, surf, ns, fmt, where, out);
}
void ll_map_release(ll_map* map) {
  if (!map) return;
  cudaSetDevice(map->device);
  for (BucketTree& t : map->tree) t.storage.release(); map->shard_owner.release(); delete map;
}
size_t ll_map_size(const ll_map* map, int which) { return map ? (size_t)map->tree[which != 0].n : 0; }

int ll_knn(ll_ctx* ctx, const ll_map* map, int which, const ll_point* queries, size_t nq, int32_t* idx5, float* sqdist5) {
  if (!ctx || !map) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  if (nq == 0) return LL_OK;
  float4* d_q; int* d_idx; float* d_d;
  LL_CUDA(ctx, ctx->feat_buf.carve([&](Carve& c) { d_q = c.take<float4>(nq); d_idx = c.take<int>(nq * LL_KNN); d_d = c.take<float>(nq * LL_KNN); }));
  LL_CUDA(ctx, cudaMemcpyAsync(d_q, queries, nq * 16, cudaMemcpyHostToDevice, ctx->stream));
  LL_TRY(launch_knn_query(ctx, map->tree[which != 0], d_q, (int)nq, d_idx, d_d));
  LL_CUDA(ctx, cudaMemcpyAsync(idx5, d_idx, nq * 20, cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaMemcpyAsync(sqdist5, d_d, nq * 20, cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return LL_OK;
}

// ---------------------------------------------------------------------------------------------- S3
static void fill_state(RegDevState* h, const ll_reg_state* in) {
  memset(h, 0, sizeof(RegDevState));
  for (int k = 0; k < 4; k++) { h->pose_curr[k] = in->q_w_curr[k]; h->pose_last[k] = in->q_w_last[k]; }
  for (int k = 0; k < 3; k++) { h->pose_curr[4 + k] = in->t_w_curr[k]; h->pose_last[4 + k] = in->t_w_last[k]; }
  for (int k = 0; k < 7; k++) h->x[k] = in->para_buffer_incremental[k];
  h->q_last_opt[0] = 1.0;
  h->bound = (double)(float)in->para_max_speed; h->huber_a = in->huber_a; h->inliner_dis = in->inliner_dis; h->inlier_ratio = in->inlier_ratio;
  h->min_icp_R = in->minimum_icp_R_diff; h->min_icp_T = in->minimum_icp_T_diff;
  h->cap = in->maximum_allow_residual_block; h->rng_seed = in->rng_seed; h->icp_max_iterations = in->icp_max_iterations;
  h->if_motion_deblur = in->if_motion_deblur ? 1 : 0; h->min_ts = in->minimum_pt_time_stamp; h->max_ts = in->maximum_pt_time_stamp;   // interp_* = 0: reset_incremtal_parameter (:120-125)
}
// The n items of a registration batch: item j's features are slots off[j] ... off[j] + nc[j] + ns[j] of A.feat (corners first), one item after
// another; its parameters in[j], its state d_reg[j].
struct RegBatch { int n; int nc[LL_MAX_BATCH], ns[LL_MAX_BATCH], off[LL_MAX_BATCH + 1]; const ll_reg_state* in[LL_MAX_BATCH]; };
static KnnBlocksArgs knn_args(ll_ctx* ctx, const ll_map* map, const RegBatch& b, bool debug) {
  const RegArrays& A = ctx->A;
  KnnBlocksArgs a; a.corner = make_view(map->tree[0]); a.surf = make_view(map->tree[1]); a.feat = A.feat; a.M = b.off[b.n]; a.n_items = b.n;
  for (int j = 0; j < b.n; j++) {
    const ll_reg_state* in = b.in[j]; KnnItem& I = a.item[j];
    I.off = b.off[j]; I.n_corner = b.nc[j]; I.n_surf = b.ns[j]; I.icp_line = in->icp_line; I.icp_plane = in->icp_plane;
    I.cap = in->maximum_allow_residual_block; I.rng_seed = in->rng_seed;
    I.max_dis_line = in->maximum_dis_line_for_match; I.max_dis_plane = in->maximum_dis_plane_for_match;
  }
  a.blk_a = A.blk_a; a.blk_v = A.blk_v;
  a.seed_ids = A.knn_idx; a.knn_d = debug ? A.knn_d : nullptr; a.perm = A.perm;
  ctx->solve_world = (map->world > 1 && ctx->world > 1) ? ctx->world : 1;   // replicas of the whole map never exchange anything
  a.st = ctx->d_reg; a.deblur = b.in[0]->if_motion_deblur ? 1 : 0; ctx->reg_deblur = a.deblur;   // (the items of a batch agree on it)
  a.rank = map->rank; a.world = map->world; a.grid = map->grid; a.shard_owner = (const int*)map->shard_owner.p;
  a.dev_counts = nullptr;
  return a;
}
static RegBatch single_batch(int nc, int ns, const ll_reg_state* in) {
  RegBatch b; b.n = 1; b.nc[0] = nc; b.ns[0] = ns; b.off[0] = 0; b.off[1] = nc + ns; b.in[0] = in;
  return b;
}
// One solver item over slots 0 ... M - 1 (the parity hooks and the sharded mode's two solves).
static SolveArgs solve_args(ll_ctx* ctx, int M, SolveMode mode, int max_iter) {
  const RegArrays& A = ctx->A;
  SolveArgs s; s.st = ctx->d_reg; s.sync = ctx->d_sync; s.feat = A.feat; s.blk_a = A.blk_a; s.blk_v = A.blk_v; s.l1 = A.l1; s.k10_value = A.k10_value; s.k10_n_distinct = A.k10_n_distinct;
  s.mode = mode; s.rank = ctx->rank; s.world = ctx->solve_world; s.comm_local = (double*)ctx->comm_local;
  for (int i = 0; i < 8; i++) s.comm_peer[i] = (double*)ctx->comm_peers[i];
  s.deblur = ctx->reg_deblur; s.n_items = 1; s.dev_counts = nullptr; s.snap = nullptr;
  SolveItem& I = s.item[0];
  I.off = 0; I.M = M; I.max_iterations = max_iter; I.prerun_iterations = 0; I.cap_check = 0; I.table = nullptr; I.table_mask = 0;
  return s;
}

}  // extern "C"

// The gate (:199): CORNER_MIN_MAP_NUM 0, SURFACE_MIN_MAP_NUM 50.
static bool reg_gate(const ll_map* map, const ll_reg_state* in) {
  return map->tree[0].n_src > 0 && map->tree[1].n_src > 50 && in->current_frame_index > in->mapping_init_accumulate_frames;
}
// What an item returns before any device work: the result initialised from its state, the gate (:199) and the empty item.  Returns 1 when the
// item goes on to the device; else *status is its outcome (LL_OK with registered = 0 under the gate, LL_ERR_NO_BLOCKS without features).
static int item_prologue(ll_ctx* ctx, const ll_map* map, int M, const ll_reg_state* in, ll_reg_result* out, int* status) {
  memset(out, 0, sizeof(*out));
  out->status = 1;
  for (int k = 0; k < 4; k++) { out->q_w_curr[k] = in->q_w_curr[k]; out->q_w_incre[k] = k == 0 ? in->para_buffer_incremental[3] : in->para_buffer_incremental[k - 1]; }
  for (int k = 0; k < 3; k++) { out->t_w_curr[k] = in->t_w_curr[k]; out->t_w_incre[k] = in->para_buffer_incremental[4 + k]; }
  *status = LL_OK;
  if (!reg_gate(map, in)) return 0;
  if (M == 0) { ctx->set_error("no features"); *status = LL_ERR_NO_BLOCKS; return 0; }
  return 1;
}

// ll_scan_to_pose's registration of the front end's features on the device counts (A.dev_counts), with no host read in between: the one item's
// slot count in the RegBatch is the capacity, and the host learns the counts at its first wait in the ICP loop.  Then, from the front end's
// counts in pinned memory: st = front_end_counts' outcome for them (LL_OK or LL_ERR_CAPACITY), nc / ns, dropped; `stopped` when the
// device counts were zero (dropped, over capacity, or no feature), so that nothing ran and the caller reports the outcome.
struct DevHandoff { const ll_pipeline_cfg* pc; int st, nc, ns, dropped, stopped; };

// The ICP loops of the batch's items on the device (every item has passed item_prologue and the capacity check): one kNN launch and one solver
// launch per ICP iteration for all of them.  outs[j] / status[j] belong to item j.  With `hand` (one item), the caller has uploaded the state.
static int register_batch(ll_ctx* ctx, const ll_map* map, const RegBatch& b, ll_reg_result* const* outs, int* const* status, DevHandoff* hand = nullptr) {
  cudaStream_t s = ctx->stream;
  const RegArrays& A = ctx->A;
  RegEvents& ev = ctx->ev;
  const int n = b.n, Mtot = b.off[n];
  if (!hand) {
    ctx->last_nc = b.nc[0]; ctx->last_ns = b.ns[0];
    RegDevState* h = ctx->pin->state_in;
    for (int j = 0; j < n; j++) fill_state(&h[j], b.in[j]);
    LL_CUDA(ctx, cudaMemcpyAsync(ctx->d_reg, h, n * sizeof(RegDevState), cudaMemcpyHostToDevice, s));
  }
  LL_CUDA(ctx, cudaEventRecord(ev.total[0], s));
  for (int j = 0; j < n; j++) outs[j]->registered = 1;
  KnnBlocksArgs ka = knn_args(ctx, map, b, false);
  if (hand) ka.dev_counts = A.dev_counts;
  LL_CUDA(ctx, cudaMemsetAsync(A.knn_idx, 0xff, (size_t)Mtot * LL_KNN * 4, s));   // no seeds for the first ICP iteration
  LL_CUDA(ctx, cudaEventRecord(ev.sort[0], s));
  LL_TRY(launch_query_sort(ctx, s, ctx->scratch, ka, A.perm));   // spatial tiles of features (Hilbert order at the initial poses)
  LL_CUDA(ctx, cudaEventRecord(ev.sort[1], s));
  int iter = 0;
  const ll_reg_state* in = b.in[0];   // the sharded mode (one item)
  const int M = Mtot;
  const bool sharded = ctx->world > 1 && map->world > 1;
  if (sharded && (map->world != ctx->world || map->rank != ctx->rank)) { ctx->set_error("map shard and context disagree on rank/world"); return LL_ERR_INVALID; }
  // (the shard was built with halo * 1.0001 + 1 mm, shard.cu: a halo handed over as the float nearest to sqrt(gate) must pass)
  if (map->world > 1 && (std::sqrt(in->maximum_dis_line_for_match) > (double)map->halo[0] * 1.0001 + 1e-3 || std::sqrt(in->maximum_dis_plane_for_match) > (double)map->halo[1] * 1.0001 + 1e-3)) {
    ctx->set_error("match gates wider than the halo this shard was built with: owner + halo search would no longer be exact"); return LL_ERR_INVALID;
  }
  if (map->world > 1 && ctx->world != map->world) { ctx->set_error("a sharded map needs a context connected to the same number of ranks (ll_comm_connect)"); return LL_ERR_INVALID; }
  if (sharded && M > ctx->cfg.max_features) { ctx->set_error("more features than max_features (exchange buffer)"); return LL_ERR_CAPACITY; }
  const int cap_check = M > in->maximum_allow_residual_block ? 1 : 0;   // fewer slots than the cap: neither the pre-skip nor the drop rule can fire
  double* x_l1 = sharded ? (double*)((char*)ctx->comm_local + LL_COMM_X_OFF) : nullptr;
  unsigned long long* set_table[LL_MAX_BATCH];   // hash set of each item's L1 norms (K10)
  LL_CUDA(ctx, ctx->scratch.carve([&](Carve& c) { for (int j = 0; j < n; j++) set_table[j] = l1_set_layout(c, b.nc[j] + b.ns[j]); }));
  // One ICP iteration's device work + a snapshot of the n 1.7 KB states into pinned slot `it & 1` (written by the fused solver launch).
  RegDevState (*slots)[LL_MAX_BATCH] = ctx->pin->snap;
  auto enqueue_iteration = [&](int it) -> int {
    cudaEvent_t* e = it < LL_TIMED_ITERS ? ev.phase[it] : nullptr;
    // corner_avail, surf_avail, n_blocks of every item: zero in the uploaded state, and cleared by the fused solver launch of every iteration
    // (SolveArgs::snap); the sharded mode clears them here
    if (sharded) LL_CUDA(ctx, cudaMemsetAsync(&ctx->d_reg->corner_avail, 0, 3 * sizeof(int), s));
    if (sharded) LL_CUDA(ctx, cudaMemsetAsync(x_l1, 0xff, (size_t)M * sizeof(double), s));   // NaN = nobody owns a block here (peers fill it after solve #1)
    if (it == 0) LL_CUDA(ctx, cudaEventRecord(ev.knn_first[0], s));
    if (e) LL_CUDA(ctx, cudaEventRecord(e[0], s));
    LL_TRY(launch_knn_blocks(ctx, ka));
    if (e) LL_CUDA(ctx, cudaEventRecord(e[1], s));
    if (it == 0) LL_CUDA(ctx, cudaEventRecord(ev.knn_first[1], s));
    if (!sharded) {
      // one launch: per item, solve #1 -> L1 norms -> de-duplication + order statistic -> outlier drop -> solve #2 -> pose
      SolveArgs sa = solve_args(ctx, M, SOLVE_FUSED, 0);
      sa.n_items = n; sa.dev_counts = ka.dev_counts; sa.snap = slots[it & 1];
      for (int j = 0; j < n; j++) {
        SolveItem& I = sa.item[j]; const int Mj = b.nc[j] + b.ns[j];
        I.off = b.off[j]; I.M = Mj; I.max_iterations = b.in[j]->cere_max_iterations; I.prerun_iterations = b.in[j]->cere_prerun_times;
        I.cap_check = Mj > b.in[j]->maximum_allow_residual_block ? 1 : 0; I.table = set_table[j]; I.table_mask = l1_set_capacity(Mj) - 1;
      }
      if (e) { LL_CUDA(ctx, cudaEventRecord(e[2], s)); LL_CUDA(ctx, cudaEventRecord(e[3], s)); }
      LL_TRY(launch_solve(ctx, sa));
    } else {
      if (cap_check) LL_TRY(launch_count_exchange(ctx));
      { SolveArgs sa = solve_args(ctx, M, SOLVE_FIRST, in->cere_prerun_times); sa.item[0].cap_check = cap_check; LL_TRY(launch_solve(ctx, sa)); }
      if (e) LL_CUDA(ctx, cudaEventRecord(e[2], s));
      LL_TRY(launch_l1_exchange(ctx, A.l1, M));
      LL_TRY(launch_k10_select(ctx, x_l1, M, &ctx->d_reg->inlier_ratio, set_table[0], l1_set_capacity(M) - 1, A.k10_value, A.k10_n_distinct));
      if (e) LL_CUDA(ctx, cudaEventRecord(e[3], s));
      { SolveArgs sa = solve_args(ctx, M, SOLVE_SECOND, in->cere_max_iterations); sa.item[0].cap_check = cap_check; LL_TRY(launch_solve(ctx, sa)); }
    }
    if (e) LL_CUDA(ctx, cudaEventRecord(e[4], s));
    if (sharded) LL_CUDA(ctx, cudaMemcpyAsync(slots[it & 1], ctx->d_reg, n * sizeof(RegDevState), cudaMemcpyDeviceToHost, s));
    LL_CUDA(ctx, cudaEventRecord(ctx->sev.it[it & 1], s));
    return LL_OK;
  };
  // The host stays one iteration ahead: iteration k+1 is enqueued before iteration k's states are read back, so the GPU never waits for the
  // PCIe round trip of the termination test.  The kernels of an iteration enqueued after an item's loop has ended return at once for that item
  // (st->icp_done: set on the device by convergence, by the item's own icp_max_iterations, or when no residual block is left).
  const bool speculate = !sharded;
  int max_iters = 0; for (int j = 0; j < n; j++) max_iters = std::max(max_iters, b.in[j]->icp_max_iterations);
  RegDevState fin[LL_MAX_BATCH];   // each item's state at the iteration its loop ended
  int done[LL_MAX_BATCH] = {0}, iters[LL_MAX_BATCH] = {0}, n_done = 0;
  LL_TRY(enqueue_iteration(0));
  for (iter = 0; iter < max_iters; iter++) {
    if (speculate && iter + 1 < max_iters) LL_TRY(enqueue_iteration(iter + 1));
    LL_CUDA(ctx, cudaEventSynchronize(ctx->sev.it[iter & 1]));
    if (hand && iter == 0) {   // the front end has completed: its counts are in pinned memory
      hand->st = front_end_counts(ctx, hand->pc, &hand->nc, &hand->ns, &hand->dropped);
      hand->stopped = hand->st != LL_OK || hand->dropped || hand->nc + hand->ns == 0;
      if (hand->stopped) break;
      ctx->last_nc = hand->nc; ctx->last_ns = hand->ns;
    }
    for (int j = 0; j < n; j++) {
      if (done[j]) continue;
      const RegDevState* hs = &slots[iter & 1][j];
      if (hs->lm.termination == -1) {
        done[j] = -1; n_done++; *status[j] = LL_ERR_NO_BLOCKS;
        ctx->set_error(n == 1 ? std::string("no residual block survived the gates / cap / inlier selection")
                              : "item " + std::to_string(j) + ": no residual block survived the gates / cap / inlier selection");
      } else if (hs->icp_done || iter + 1 >= b.in[j]->icp_max_iterations) { done[j] = 1; n_done++; fin[j] = *hs; iters[j] = iter + 1; }
    }
    if (n_done == n) break;
    if (!speculate && iter + 1 < max_iters) LL_TRY(enqueue_iteration(iter + 1));
  }
  // (an iteration enqueued ahead returns at once; it is drained here, before the arena is reused)
  LL_CUDA(ctx, cudaEventRecord(ev.total[1], s));
  LL_CUDA(ctx, cudaEventSynchronize(ev.total[1]));
  if (hand && hand->stopped) return LL_OK;
  ll_reg_result t; memset(&t, 0, sizeof(t));   // the batch's timings, given to every item
  cudaEventElapsedTime(&t.gpu_ms_total, ev.total[0], ev.total[1]); cudaEventElapsedTime(&t.gpu_ms_knn, ev.knn_first[0], ev.knn_first[1]);
  cudaEventElapsedTime(&t.gpu_ms_sort, ev.sort[0], ev.sort[1]);
  { const int done_iters = (iter < max_iters ? iter + 1 : max_iters);
    for (int i = 0; i < done_iters && i < LL_TIMED_ITERS; i++) { float a = 0, b = 0, c = 0, d = 0; cudaEvent_t* e = ev.phase[i];
      cudaEventElapsedTime(&a, e[0], e[1]); cudaEventElapsedTime(&b, e[1], e[2]); cudaEventElapsedTime(&c, e[2], e[3]); cudaEventElapsedTime(&d, e[3], e[4]);
      t.gpu_ms_knn_all += a; t.gpu_ms_solve_all += b + d; t.gpu_ms_select_all += c; } }
  for (int j = 0; j < n; j++) {
    if (done[j] != 1) continue;
    const RegDevState* hs = &fin[j]; const ll_reg_state* in = b.in[j]; ll_reg_result* out = outs[j];
    out->gpu_ms_total = t.gpu_ms_total; out->gpu_ms_knn = t.gpu_ms_knn; out->gpu_ms_sort = t.gpu_ms_sort;
    out->gpu_ms_knn_all = t.gpu_ms_knn_all; out->gpu_ms_solve_all = t.gpu_ms_solve_all; out->gpu_ms_select_all = t.gpu_ms_select_all;
    out->icp_iterations = iters[j];
    out->corner_used = hs->corner_avail; out->surf_used = hs->surf_avail; out->num_residual_blocks = hs->num_residual_blocks;
    out->total_lm_iterations = hs->total_lm_iterations; out->total_evaluations = hs->total_evaluations;
    for (int k = 0; k < 4; k++) out->q_w_curr[k] = hs->pose_curr[k];
    for (int k = 0; k < 3; k++) out->t_w_curr[k] = hs->pose_curr[4 + k];
    out->q_w_incre[0] = hs->x[3]; out->q_w_incre[1] = hs->x[0]; out->q_w_incre[2] = hs->x[1]; out->q_w_incre[3] = hs->x[2];
    for (int k = 0; k < 3; k++) out->t_w_incre[k] = hs->x[4 + k];
    out->final_cost = hs->final_cost; out->initial_cost = hs->initial_cost; out->angular_diff = hs->angular_diff; out->t_diff = hs->t_diff;
    out->inlier_threshold = hs->inlier_threshold * hs->final_cost / hs->initial_cost;   // :559
    const float minimize_cost = (float)hs->final_cost;
    if (hs->angular_diff > (double)(float)in->para_max_angular_rate || minimize_cost > (float)in->max_final_cost) {   // :561-573
      out->status = 0;
      for (int k = 0; k < 4; k++) out->q_w_curr[k] = in->q_w_last[k];
      for (int k = 0; k < 3; k++) out->t_w_curr[k] = in->t_w_last[k];
    }
  }
  return LL_OK;
}

int register_device(ll_ctx* ctx, const ll_map* map, int nc, int ns, const ll_reg_state* in, ll_reg_result* out) {
  int st = LL_OK;
  if (!item_prologue(ctx, map, nc + ns, in, out, &st)) {
    if (st != LL_OK) { ctx->last_nc = 0; ctx->last_ns = 0; }   // an empty registration has no features
    return st;
  }
  const int M = nc + ns;
  LL_TRY(solve_capacity(ctx, 1, &M, in->if_motion_deblur ? 1 : 0));   // before anything of this registration is enqueued
  int* stp = &st;
  LL_TRY(register_batch(ctx, map, single_batch(nc, ns, in), &out, &stp));
  return st;
}

int features_fit(ll_ctx* ctx, size_t nc, size_t ns) {
  if (nc + ns <= (size_t)ctx->cfg.max_features) return LL_OK;
  ctx->set_error("more features than max_features"); return LL_ERR_CAPACITY;
}

int features_hand_over(ll_ctx* ctx, cudaStream_t s, const float4* corner, int nc, const float4* surf, int ns) {
  LL_CUDA(ctx, cudaMemcpyAsync(ctx->A.feat, corner, (size_t)nc * 16, cudaMemcpyDeviceToDevice, s));
  LL_CUDA(ctx, cudaMemcpyAsync(ctx->A.feat + nc, surf, (size_t)ns * 16, cudaMemcpyDeviceToDevice, s));
  return LL_OK;
}

extern "C" {

int ll_register(ll_ctx* ctx, const ll_map* map, const void* scan_corner, size_t nc, const void* scan_surf, size_t ns, int fmt, int where, const ll_reg_state* in, ll_reg_result* out) {
  if (!ctx || !map || !in || !out) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  LL_TRY(features_fit(ctx, nc, ns));
  LL_TRY(upload_cloud(ctx, ctx->stream, scan_corner, nc, fmt, where, ctx->A.feat));
  LL_TRY(upload_cloud(ctx, ctx->stream, scan_surf, ns, fmt, where, ctx->A.feat + nc));
  return register_device(ctx, map, (int)nc, (int)ns, in, out);
}

int ll_register_batch(ll_ctx* ctx, const ll_map* map, int n, const void* const* corners, const size_t* n_corner, const void* const* surfs, const size_t* n_surf,
                      int fmt, int where, const ll_reg_state* in, ll_reg_result* out, int* item_status) {
  if (!ctx || !map || !corners || !n_corner || !surfs || !n_surf || !in || !out || !item_status) return LL_ERR_INVALID;
  if (n < 1 || n > LL_MAX_BATCH) { ctx->set_error("n = " + std::to_string(n) + ": a batch holds 1 ... " + std::to_string(LL_MAX_BATCH) + " items"); return LL_ERR_INVALID; }
  if (map->world > 1) { ctx->set_error("a sharded map registers one scan at a time (ll_register)"); return LL_ERR_INVALID; }
  cudaSetDevice(ctx->device);
  size_t total = 0;
  for (int i = 0; i < n; i++) {
    if ((!corners[i] && n_corner[i]) || (!surfs[i] && n_surf[i])) { ctx->set_error("item " + std::to_string(i) + ": null feature cloud"); return LL_ERR_INVALID; }
    if ((in[i].if_motion_deblur != 0) != (in[0].if_motion_deblur != 0)) { ctx->set_error("item " + std::to_string(i) + ": if_motion_deblur differs from item 0's"); return LL_ERR_INVALID; }
    total += n_corner[i] + n_surf[i];
  }
  if (total > (size_t)ctx->cfg.max_features) { ctx->set_error("the items' features (" + std::to_string(total) + ") exceed max_features"); return LL_ERR_CAPACITY; }
  // the items that go on to the device, their features one after another
  RegBatch b; b.n = 0; b.off[0] = 0;
  int idx[LL_MAX_BATCH], M[LL_MAX_BATCH];
  for (int i = 0; i < n; i++) {
    if (!item_prologue(ctx, map, (int)(n_corner[i] + n_surf[i]), &in[i], &out[i], &item_status[i])) continue;
    const int j = b.n++;
    idx[j] = i; b.nc[j] = (int)n_corner[i]; b.ns[j] = (int)n_surf[i]; b.in[j] = &in[i]; M[j] = b.nc[j] + b.ns[j]; b.off[j + 1] = b.off[j] + M[j];
  }
  if (b.n == 0) return LL_OK;
  int bad = 0;
  if (solve_capacity(ctx, b.n, M, in[0].if_motion_deblur ? 1 : 0, &bad) != LL_OK) { ctx->set_error("item " + std::to_string(idx[bad]) + ": " + ctx->err); return LL_ERR_CAPACITY; }
  for (int j = 0; j < b.n; j++) {
    LL_TRY(upload_cloud(ctx, ctx->stream, corners[idx[j]], b.nc[j], fmt, where, ctx->A.feat + b.off[j]));
    LL_TRY(upload_cloud(ctx, ctx->stream, surfs[idx[j]], b.ns[j], fmt, where, ctx->A.feat + b.off[j] + b.nc[j]));
  }
  ll_reg_result* outs[LL_MAX_BATCH]; int* sts[LL_MAX_BATCH];
  for (int j = 0; j < b.n; j++) { outs[j] = &out[idx[j]]; sts[j] = &item_status[idx[j]]; }
  return register_batch(ctx, map, b, outs, sts);
}

// One tiny registration (three planes and two edges: 1240 map points, 310 features) through the whole device path, result discarded.  It pays -- once, at a
// time of the caller's choosing -- what CUDA defers to first use: the module loads of the kNN / solver / sort kernels and the first cooperative launch
// (otherwise paid by the first registered scan of a stream).  ll_mapper_create calls it.
int ll_ctx_warmup(ll_ctx* ctx) {
  if (!ctx) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  std::vector<ll_point> surf, corner, fs, fc;
  auto add = [](std::vector<ll_point>& v, float x, float y, float z) { ll_point p; p.x = x; p.y = y; p.z = z; p.intensity = 0.f; v.push_back(p); };
  for (int i = 0; i < 20; i++) for (int j = 0; j < 20; j++) {
    const float u = 0.1f * i + 0.013f * (j % 3), v = 0.1f * j + 0.007f * (i % 5);
    add(surf, 1.f + u, -1.f + v, 0.f); add(surf, 1.f + u, 1.2f, 0.05f + v); add(surf, 3.2f, -1.f + u, 0.05f + v);
    if ((i * 20 + j) % 4 == 0) { add(fs, 1.f + u + 0.004f, -1.f + v - 0.003f, 0.006f); add(fs, 1.f + u, 1.195f, 0.05f + v); add(fs, 3.194f, -1.f + u, 0.05f + v); }
  }
  for (int k = 0; k < 20; k++) { add(corner, 3.2f, 1.2f, 0.1f * k); add(corner, 1.f + 0.1f * k, 1.2f, 0.f); if (k % 4 == 0) { add(fc, 3.195f, 1.197f, 0.1f * k + 0.02f); add(fc, 1.02f + 0.1f * k, 1.196f, 0.004f); } }
  if ((int)(fc.size() + fs.size()) > ctx->cfg.max_features) return LL_OK;   // a context sized for less than the toy problem: nothing to warm
  ll_map* m = nullptr;
  int st = ll_map_build(ctx, corner.data(), corner.size(), surf.data(), surf.size(), LL_FMT_XYZI16, LL_HOST, &m);
  if (st == LL_OK) {
    ll_reg_state rs; ll_reg_state_default(&rs); rs.current_frame_index = rs.mapping_init_accumulate_frames + 1;
    ll_reg_result r;
    st = ll_register(ctx, m, fc.data(), fc.size(), fs.data(), fs.size(), LL_FMT_XYZI16, LL_HOST, &rs, &r);
    if (st == LL_ERR_NO_BLOCKS) st = LL_OK;   // (nothing here depends on the outcome of the toy problem)
  }
  if (m) ll_map_release(m);
  if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) return LL_ERR_CUDA;
  return st;
}

int ll_build_blocks(ll_ctx* ctx, const ll_map* map, const void* scan_corner, size_t nc, const void* scan_surf, size_t ns, int fmt, int where, const ll_reg_state* in,
                    int32_t* type, double* a3, double* v3, int* corner_avail, int* surf_avail) {
  if (!ctx || !map || !in) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  const int M = (int)(nc + ns);
  if (M > ctx->cfg.max_features) return LL_ERR_CAPACITY;
  const RegArrays& A = ctx->A;
  cudaStream_t s = ctx->stream;
  LL_TRY(upload_cloud(ctx, ctx->stream, scan_corner, nc, fmt, where, A.feat));
  LL_TRY(upload_cloud(ctx, ctx->stream, scan_surf, ns, fmt, where, A.feat + nc));
  RegDevState* h = ctx->pin->state_in; fill_state(h, in);
  LL_CUDA(ctx, cudaMemcpyAsync(ctx->d_reg, h, sizeof(RegDevState), cudaMemcpyHostToDevice, s));
  { KnnBlocksArgs ka = knn_args(ctx, map, single_batch((int)nc, (int)ns, in), true); LL_CUDA(ctx, cudaMemsetAsync(A.knn_idx, 0xff, (size_t)M * LL_KNN * 4, s)); LL_TRY(launch_query_sort(ctx, s, ctx->scratch, ka, A.perm)); LL_TRY(launch_knn_blocks(ctx, ka)); }
  std::vector<float4> ba(M); std::vector<double> bv((size_t)M * 3);
  int cnt[2];
  LL_CUDA(ctx, cudaMemcpyAsync(ba.data(), A.blk_a, (size_t)M * 16, cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaMemcpyAsync(bv.data(), A.blk_v, (size_t)M * 24, cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaMemcpyAsync(cnt, &ctx->d_reg->corner_avail, 8, cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  for (int i = 0; i < M; i++) {
    int t; memcpy(&t, &ba[i].w, 4);
    if (type) type[i] = t;
    if (a3) { a3[3 * i] = ba[i].x; a3[3 * i + 1] = ba[i].y; a3[3 * i + 2] = ba[i].z; }
    if (v3) { v3[3 * i] = bv[3 * i]; v3[3 * i + 1] = bv[3 * i + 1]; v3[3 * i + 2] = bv[3 * i + 2]; }
  }
  if (corner_avail) *corner_avail = cnt[0]; if (surf_avail) *surf_avail = cnt[1];
  ctx->hook_slots = M;   // slot count for ll_normal_equations / ll_solve
  return LL_OK;
}
}  // extern "C"

// The solver parity hooks: x to the device state, one solver launch over the hook's slots, the state back into snap[0] (and the L1 norms
// into l1_out when given), then synchronise.
static int hook_solve(ll_ctx* ctx, const double x[7], const SolveArgs& sa, double* l1_out = nullptr) {
  cudaStream_t s = ctx->stream;
  PinnedStage* pin = ctx->pin;
  for (int k = 0; k < 7; k++) pin->x[k] = x[k];
  LL_CUDA(ctx, cudaMemcpyAsync(ctx->d_reg->x, pin->x, 7 * sizeof(double), cudaMemcpyHostToDevice, s));
  LL_TRY(launch_solve(ctx, sa));
  LL_CUDA(ctx, cudaMemcpyAsync(&pin->snap[0][0], ctx->d_reg, sizeof(RegDevState), cudaMemcpyDeviceToHost, s));
  if (l1_out && sa.item[0].M > 0) LL_CUDA(ctx, cudaMemcpyAsync(l1_out, ctx->A.l1, (size_t)sa.item[0].M * sizeof(double), cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  return LL_OK;
}

extern "C" {

int ll_normal_equations(ll_ctx* ctx, const double x[7], double out28[28]) {
  if (!ctx || !x || !out28) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  LL_TRY(hook_solve(ctx, x, solve_args(ctx, ctx->hook_slots, SOLVE_EVALUATE, 0)));
  const RegDevState* hs = &ctx->pin->snap[0][0];
  for (int i = 0; i < 21; i++) out28[i] = hs->lm.H[i];
  for (int i = 0; i < 6; i++) out28[21 + i] = hs->lm.g[i];
  out28[27] = hs->lm.x_cost;
  return LL_OK;
}
int ll_solve(ll_ctx* ctx, int max_iterations, double x_io[7], double* initial_cost, double* final_cost, int* iterations) {
  if (!ctx || !x_io) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  LL_TRY(hook_solve(ctx, x_io, solve_args(ctx, ctx->hook_slots, SOLVE_PLAIN, max_iterations)));
  const RegDevState* hs = &ctx->pin->snap[0][0];
  for (int k = 0; k < 7; k++) x_io[k] = hs->x[k];
  if (initial_cost) *initial_cost = hs->lm.initial_cost; if (final_cost) *final_cost = hs->lm.final_cost; if (iterations) *iterations = hs->lm.iteration;
  return LL_OK;
}
int ll_set_blocks(ll_ctx* ctx, const ll_reg_state* in, size_t n, const int32_t* type, const ll_point* p, const float* a3, const double* v3) {
  if (!ctx || !in || (n > 0 && (!type || !p || !a3 || !v3))) return LL_ERR_INVALID;
  if (n > (size_t)ctx->cfg.max_features) { ctx->set_error("more blocks than max_features"); return LL_ERR_CAPACITY; }
  const int M = (int)n;
  LL_TRY(solve_capacity(ctx, 1, &M, in->if_motion_deblur ? 1 : 0));
  for (int i = 0; i < M; i++) if (type[i] < 0 || type[i] > 2) { ctx->set_error("block type must be 0, 1 (line) or 2 (plane)"); return LL_ERR_INVALID; }
  cudaSetDevice(ctx->device);
  const RegArrays& A = ctx->A;
  cudaStream_t s = ctx->stream;
  std::vector<float4> ba(M);
  for (int i = 0; i < M; i++) { ba[i].x = a3[3 * i]; ba[i].y = a3[3 * i + 1]; ba[i].z = a3[3 * i + 2]; memcpy(&ba[i].w, &type[i], 4); }
  if (M > 0) {
    LL_CUDA(ctx, cudaMemcpyAsync(A.feat, p, (size_t)M * 16, cudaMemcpyHostToDevice, s));
    LL_CUDA(ctx, cudaMemcpyAsync(A.blk_a, ba.data(), (size_t)M * 16, cudaMemcpyHostToDevice, s));
    LL_CUDA(ctx, cudaMemcpyAsync(A.blk_v, v3, (size_t)M * 24, cudaMemcpyHostToDevice, s));
  }
  RegDevState* h = ctx->pin->state_in; fill_state(h, in);
  for (int i = 0; i < M; i++) h->n_blocks += type[i] != 0 ? 1 : 0;   // what the kNN kernel counts: the drop rule of the residual-block cap reads it
  LL_CUDA(ctx, cudaMemcpyAsync(ctx->d_reg, h, sizeof(RegDevState), cudaMemcpyHostToDevice, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));   // the pageable staging above goes out of scope
  ctx->hook_slots = M; ctx->hook_cap_check = M > in->maximum_allow_residual_block ? 1 : 0;
  ctx->reg_deblur = in->if_motion_deblur ? 1 : 0; ctx->solve_world = 1;
  return LL_OK;
}
int ll_solve_fused(ll_ctx* ctx, int prerun, int max_iterations, double x_io[7], double* threshold, int* n_distinct, int* n_kept, double* l1_out, int iterations[2]) {
  if (!ctx || !x_io) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  const int M = ctx->hook_slots;
  cudaStream_t s = ctx->stream;
  SolveArgs sa = solve_args(ctx, M, SOLVE_FUSED, max_iterations);
  SolveItem& I = sa.item[0];
  LL_CUDA(ctx, ctx->scratch.carve([&](Carve& c) { I.table = l1_set_layout(c, M); }));
  I.prerun_iterations = prerun; I.table_mask = l1_set_capacity(M) - 1;
  I.cap_check = ctx->hook_cap_check;
  // a fused launch ends with the ICP termination test: the flag and the iteration totals start afresh for every call
  LL_CUDA(ctx, cudaMemsetAsync(&ctx->d_reg->icp_done, 0, sizeof(int), s));
  LL_CUDA(ctx, cudaMemsetAsync(&ctx->d_reg->total_lm_iterations, 0, 2 * sizeof(int), s));   // total_lm_iterations, total_evaluations
  LL_TRY(hook_solve(ctx, x_io, sa, l1_out));
  const RegDevState* hs = &ctx->pin->snap[0][0];
  for (int k = 0; k < 7; k++) x_io[k] = hs->x[k];
  if (threshold) *threshold = hs->inlier_threshold; if (n_distinct) *n_distinct = hs->n_unique; if (n_kept) *n_kept = hs->num_residual_blocks;
  if (iterations) { iterations[1] = hs->lm.iteration; iterations[0] = hs->total_lm_iterations - hs->lm.iteration; }
  return LL_OK;
}
int ll_inlier_select(ll_ctx* ctx, const double* l1, size_t n, double ratio, double* value, int* n_distinct) {
  if (!ctx || (n > 0 && !l1) || !value || !n_distinct || !(ratio >= 0.0)) return LL_ERR_INVALID;
  for (size_t i = 0; i < n; i++) if (l1[i] < 0.0) { ctx->set_error("L1 norms are never negative"); return LL_ERR_INVALID; }
  if (n > (size_t)ctx->cfg.max_features) { ctx->set_error("more values than max_features"); return LL_ERR_CAPACITY; }
  cudaSetDevice(ctx->device);
  const int M = (int)n;
  const RegArrays& A = ctx->A;
  cudaStream_t s = ctx->stream;
  if (M > 0) LL_CUDA(ctx, cudaMemcpyAsync(A.l1, l1, n * sizeof(double), cudaMemcpyHostToDevice, s));
  double* d_ratio = &ctx->d_reg->inlier_ratio;   // read on the device as a registration reads it (ll_register rewrites the whole state)
  LL_CUDA(ctx, cudaMemcpyAsync(d_ratio, &ratio, sizeof(double), cudaMemcpyHostToDevice, s));
  unsigned long long* table = nullptr;
  LL_CUDA(ctx, ctx->scratch.carve([&](Carve& c) { table = l1_set_layout(c, M); }));
  LL_TRY(launch_k10_select(ctx, A.l1, M, d_ratio, table, l1_set_capacity(M) - 1, A.k10_value, A.k10_n_distinct));
  LL_CUDA(ctx, cudaMemcpyAsync(value, A.k10_value, sizeof(double), cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaMemcpyAsync(n_distinct, A.k10_n_distinct, sizeof(int), cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  return LL_OK;
}

int ll_set_point_layout(ll_ctx* ctx, const ll_point_layout* L) {
  if (!ctx || !L) return LL_ERR_INVALID;
  const int isz = L->intensity_datatype == LL_I_FLOAT32 ? 4 : L->intensity_datatype == LL_I_UINT16 ? 2 : L->intensity_datatype == LL_I_UINT8 ? 1 : 0;
  if (L->intensity_datatype != LL_I_NONE && isz == 0) { ctx->set_error("unsupported intensity datatype"); return LL_ERR_INVALID; }
  const int offs[3] = {L->offset_x, L->offset_y, L->offset_z};
  for (int k = 0; k < 3; k++) if (offs[k] < 0 || offs[k] + 4 > L->point_step) { ctx->set_error("field outside the point record"); return LL_ERR_INVALID; }
  if (isz && (L->offset_intensity < 0 || L->offset_intensity + isz > L->point_step)) { ctx->set_error("intensity outside the point record"); return LL_ERR_INVALID; }
  ctx->layout = *L;
  return LL_OK;
}
// pcl::toROSMsg for the feature clouds the feature node publishes (laser_feature_extractor.hpp:367-384): the features of the last ll_scan_to_pose /
// ll_register / ll_frame_to_pose on this context (which = 0 corners, 1 surfaces; scan frame) as PointCloud2 records in the layout of ll_set_point_layout.
int ll_features_to_pointcloud2(ll_ctx* ctx, int which, void* out_host, size_t cap_bytes, size_t* n_points) {
  if (!ctx || !n_points || (which != 0 && which != 1)) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  const RegArrays& A = ctx->A;
  const int n = which == 0 ? ctx->last_nc : ctx->last_ns;
  const float4* src = which == 0 ? A.feat : A.feat + ctx->last_nc;
  *n_points = (size_t)n;
  const size_t bytes = (size_t)n * (size_t)ctx->layout.point_step;
  if (!out_host || n == 0) return LL_OK;
  if (cap_bytes < bytes) { ctx->set_error("output buffer smaller than n * point_step"); return LL_ERR_CAPACITY; }
  LL_CUDA(ctx, ctx->stage_in.reserve(bytes));
  LL_TRY(launch_pack_strided(ctx, src, n, ctx->stage_in.as<unsigned char>()));
  LL_CUDA(ctx, cudaMemcpyAsync(out_host, ctx->stage_in.p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return LL_OK;
}
int ll_format_pose_log(const ll_reg_result* r, char* buf, size_t cap) {
  if (!r || !buf) return -1;
  const int n = snprintf(buf, cap, "--------------------\nCurr_Q = %f,%f,%f,%f\r\nCurr_T = %f,%f,%f\r\nIncre_Q = %f,%f,%f,%f\r\nIncre_T = %f,%f,%f\r\nCost=%f,blk_size = %d \r\n",
                         r->q_w_curr[0], r->q_w_curr[1], r->q_w_curr[2], r->q_w_curr[3], r->t_w_curr[0], r->t_w_curr[1], r->t_w_curr[2],
                         r->q_w_incre[0], r->q_w_incre[1], r->q_w_incre[2], r->q_w_incre[3], r->t_w_incre[0], r->t_w_incre[1], r->t_w_incre[2],
                         r->final_cost, r->num_residual_blocks);
  return (n < 0 || (size_t)n >= cap) ? -1 : n;
}
// Bytes read back per ICP iteration (the device-side registration state snapshot): what bench.py counts as d2h traffic.
int ll_state_snapshot_bytes(void) { return (int)sizeof(RegDevState); }
// Diagnostics: the master CTA's cycle counters of the last registration (kernels.cuh: RegDevState::prof).
int ll_debug_solver_cycles(ll_ctx* ctx, long long out8[16]) {
  if (!ctx || !out8) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  LL_CUDA(ctx, cudaMemcpyAsync(out8, ctx->d_reg->prof, 16 * sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return LL_OK;
}

// ---------------------------------------------------------------------------------------------- whole per-scan step
}  // extern "C"

// Laser_feature::laserCloudHandler for one frame, on the device: extraction, piece bounds, get_features, the extractor's VoxelGrids
// (laser_feature_extractor.hpp:285-380) and the mapping node's input VoxelGrids (laser_mapping.hpp:1367-1373).  Leaves the features in
// A.feat (corners then surfaces).  *dropped = 1 when the frame has <= 5 petals (:287).
// The four VoxelGrids of a frame's features (laser_feature_extractor.hpp:372-380 then laser_mapping.hpp:1367-1373): the corner chain
// tmp_a -> tmp_d -> tmp_a, the surface chain tmp_b -> tmp_c -> tmp_b, as one cluster launch on fs.main when they fit (launch_voxel_chains),
// else the corner chain on fs.corner (fe_corner) and the surface chain on fs.main (fe_main).  The input counts are nc_cap / ns_cap, or the
// device counts d_nc / d_ns when given; the outputs land in counts[4..7].
static int voxel_chains(ll_ctx* ctx, const FrontStreams& fs, const ll_pipeline_cfg* pc, int nc_cap, const int* d_nc, int ns_cap, const int* d_ns) {
  const RegArrays& A = ctx->A; int* cnt = A.counts;
  const VgChain c[2] = {
      {{A.tmp_a, nc_cap, d_nc, 2, {pc->extractor_leaf_corner, pc->mapping_leaf_corner}, {A.tmp_d, A.tmp_a}, {cnt + 4, cnt + 5}}, &ctx->fe_corner, fs.corner},
      {{A.tmp_b, ns_cap, d_ns, 2, {pc->extractor_leaf_surf, pc->mapping_leaf_surf}, {A.tmp_c, A.tmp_b}, {cnt + 6, cnt + 7}}, &ctx->fe_main, fs.main}};
  return launch_voxel_chains(ctx, fs.main, c, 2, fs.fork, fs.join);
}

// The front end's counts and the extractor's meta into pinned memory, where front_end_counts reads them.
static int front_end_counts_d2h(ll_ctx* ctx, cudaStream_t s) {
  LL_CUDA(ctx, cudaMemcpyAsync(ctx->pin->fe_counts, ctx->A.counts, sizeof(ctx->pin->fe_counts), cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaMemcpyAsync(ctx->pin->fe_meta, ctx->ex.d_meta, sizeof(ctx->pin->fe_meta), cudaMemcpyDeviceToHost, s));
  return LL_OK;
}

// Everything of the front end that is enqueued on the device, in the order the reference runs it; counts land in pinned memory.
static int front_end_enqueue(ll_ctx* ctx, const FrontStreams& fs, const ll_pipeline_cfg* pc, int ncap) {
  cudaStream_t s = fs.main;
  const RegArrays& A = ctx->A;
  const bool petals_aside = pc->whole_frame && ctx->ex.n >= 5;   // nothing downstream of get_features reads the petal bookkeeping then
  if (petals_aside) {
    LL_TRY(launch_extract_points(ctx, s, ctx->ex.n));
    LL_CUDA(ctx, cudaEventRecord(fs.fork3, s));
    LL_CUDA(ctx, cudaStreamWaitEvent(fs.petals, fs.fork3, 0));
    LL_TRY(launch_extract_petals(ctx, ctx->ex.n, fs.petals, ctx->fe_petals));
    LL_CUDA(ctx, cudaEventRecord(fs.join3, fs.petals));
  } else LL_TRY(extract_enqueue(ctx, s, ctx->fe_main));
  const float* d_bounds = nullptr;
  if (!pc->whole_frame) { LL_TRY(launch_piece_bounds(ctx, s, pc->pieces, A.bounds)); d_bounds = A.bounds + 2 * pc->use_piece; }
  LL_TRY(launch_get_features(ctx, s, ctx->fe_main, d_bounds, 0.f, 1.f, A.tmp_a, A.tmp_b, nullptr, A.counts));
  LL_TRY(voxel_chains(ctx, fs, pc, ncap, A.counts + 0, ncap, A.counts + 1));   // counts: [0] corners [1] surf [2] full
  if (petals_aside) LL_CUDA(ctx, cudaStreamWaitEvent(s, fs.join3, 0));
  // [10], [11]: min / max time stamp of the full cloud
  return front_end_counts_d2h(ctx, s);
}

// `enqueue` (the device part of a front end, on stream s) eagerly on the first call with `key`, captured into g on the second when `capturable`,
// replayed from the third.  The graph is captured from, and replayed on, whichever streams the caller passes: it holds its own dependencies,
// so one cache serves both the single-input calls and the sequence calls.
template <typename F>
static int front_graph(ll_ctx* ctx, FrontGraph& g, cudaStream_t s, const FrontKey& key, bool capturable, F&& enqueue) {
  const bool same = g.key == key;
  if (same && g.exec) {
    LL_CUDA(ctx, cudaGraphLaunch(g.exec, s));
    ctx->launches += g.launches;
    return LL_OK;
  }
  if (same && g.warm && capturable) {
    const uint64_t l0 = ctx->launches;
    cudaGraph_t graph = nullptr;
    LL_CUDA(ctx, cudaStreamBeginCapture(s, cudaStreamCaptureModeRelaxed));
    const int st = enqueue();
    cudaError_t ce = cudaStreamEndCapture(s, &graph);
    if (st == LL_OK && ce == cudaSuccess) ce = cudaGraphInstantiate(&g.exec, graph, 0);
    if (graph) cudaGraphDestroy(graph);
    if (st == LL_OK && ce == cudaSuccess) {
      g.launches = ctx->launches - l0;
      LL_CUDA(ctx, cudaGraphLaunch(g.exec, s));
      return LL_OK;
    }
    // should not happen: the captured launches never ran, so they are not counted; eager launches, and the shape starts afresh
    cudaGetLastError(); g.exec = nullptr; ctx->launches = l0; g.warm = false; g.key = FrontKey();
    return enqueue();
  }
  if (g.exec) { cudaGraphExecDestroy(g.exec); g.exec = nullptr; }
  LL_TRY(enqueue());
  g.key = key; g.warm = true;
  return LL_OK;
}

int scan_front_end_enqueue(ll_ctx* ctx, const FrontStreams& fs, const void* raw, size_t n, int fmt, int where, double stamp, const ll_pipeline_cfg* pc) {
  LL_TRY(extract_prepare(ctx, fs.main, raw, n, fmt, where, stamp));
  FrontKey key; key.n_heads = 1; key.ns[0] = n; key.pc = *pc;
  return front_graph(ctx, ctx->fg, fs.main, key, n >= 5, [&] { return front_end_enqueue(ctx, fs, pc, (int)n); });
}

int front_end_counts(ll_ctx* ctx, const ll_pipeline_cfg* pc, int* nc_out, int* ns_out, int* dropped) {
  const int* h = ctx->pin->fe_counts;
  const int nc = h[5], ns = h[7], meta_scans = ctx->pin->fe_meta[1];
  ctx->last_full_min_t = ll_ord2f(h[10]); ctx->last_full_max_t = ll_ord2f(h[11]);
  *nc_out = nc; *ns_out = ns;
  *dropped = (meta_scans <= 5 && !pc->whole_frame) ? 1 : 0;
  if (*dropped) return LL_OK;
  return features_fit(ctx, nc, ns);
}

int scan_front_end(ll_ctx* ctx, const void* raw, size_t n, int fmt, int where, double stamp, const ll_pipeline_cfg* pc, int* nc_out, int* ns_out, int* dropped) {
  LL_TRY(scan_front_end_enqueue(ctx, ctx->own_front(), raw, n, fmt, where, stamp, pc));
  LL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  LL_TRY(front_end_counts(ctx, pc, nc_out, ns_out, dropped));
  if (*dropped) return LL_OK;
  return features_hand_over(ctx, ctx->stream, ctx->A.tmp_a, *nc_out, ctx->A.tmp_b, *ns_out);
}

// The front end's features into A.feat on the device: corners (counts[5], from tmp_a) then surfaces (counts[7], from tmp_b), and the counts
// the registration reads, dc = {corners, surfaces}.  dc = {0, 0} and nothing is copied when the frame is dropped (meta[1] <= 5 petals and not
// whole_frame, :287) or has more features than max_features: front_end_counts' rules.
__global__ void feature_handoff_kernel(const int* __restrict__ counts, const int* __restrict__ meta, int whole_frame, int max_features, const float4* __restrict__ corner,
                                       const float4* __restrict__ surf, float4* __restrict__ feat, int* __restrict__ dc) {
  const int nc = counts[5], ns = counts[7];
  const bool keep = !(meta[1] <= 5 && !whole_frame) && nc + ns <= max_features;
  if (blockIdx.x == 0 && threadIdx.x == 0) { dc[0] = keep ? nc : 0; dc[1] = keep ? ns : 0; }
  if (!keep) return;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nc + ns; i += gridDim.x * blockDim.x) feat[i] = i < nc ? corner[i] : surf[i - nc];
}

// ll_scan_to_pose without a host read between the front end and the registration: the state goes up before the front end, the features move
// into A.feat and the spatial sort and the first two ICP iterations are enqueued behind the front end at once, all sized for max_features and
// reading the counts on the device; the host reads the counts at its first wait in the ICP loop.  The outcomes and the results are those of
// the host-sized path (scan_front_end + register_device), which is taken instead when the capacity does not bound the feature count
// (max_features < max_scan_points), when the solver's shared memory cannot hold max_features slots, for a sharded map or context, under
// the gate (:199), where no registration runs, and with no ICP iteration to read the counts at.
static bool device_handoff(ll_ctx* ctx, const ll_map* map, const ll_reg_state* in) {
  if (ctx->cfg.max_features < ctx->cfg.max_scan_points || ctx->world > 1 || map->world > 1 || !reg_gate(map, in) || in->icp_max_iterations < 1) return false;
  const std::string err = ctx->err;
  if (solve_capacity(ctx, 1, &ctx->cfg.max_features, in->if_motion_deblur ? 1 : 0) != LL_OK) { ctx->err = err; return false; }
  return true;
}
// The registration on the device counts (device_handoff has passed): the state goes up, `front` enqueues what leaves the features in tmp_a /
// tmp_b, their counts in counts[5] / [7] and those on their way into pin->fe_counts / fe_meta (front_end_enqueue's end), then the hand-over,
// the registration and the outcome.  ll_scan_to_pose runs the front end here, ll_register_dev_counts uploads caller-given features.
template <typename F>
static int register_dev_counts(ll_ctx* ctx, const ll_map* map, const ll_pipeline_cfg* pc, const ll_reg_state* in, ll_reg_result* out, int* nc, int* ns,
                               int* dropped, F&& front) {
  cudaStream_t s = ctx->stream;
  const RegArrays& A = ctx->A;
  const int cap = ctx->cfg.max_features;
  RegDevState* h = ctx->pin->state_in; fill_state(h, in);
  LL_CUDA(ctx, cudaMemcpyAsync(ctx->d_reg, h, sizeof(RegDevState), cudaMemcpyHostToDevice, s));
  LL_TRY(front());
  feature_handoff_kernel<<<ctx->num_sms * 2, 256, 0, s>>>(A.counts, ctx->ex.d_meta, pc->whole_frame, cap, A.tmp_a, A.tmp_b, A.feat, A.dev_counts); ctx->launches++;
  LL_CUDA(ctx, cudaGetLastError());
  int st = LL_OK;
  item_prologue(ctx, map, cap, in, out, &st);   // (the gate has passed and cap > 0: the result initialised from the state)
  DevHandoff hand = {pc, LL_OK, 0, 0, 0, 0};
  int* stp = &st;
  LL_TRY(register_batch(ctx, map, single_batch(cap, 0, in), &out, &stp, &hand));
  *nc = hand.nc; *ns = hand.ns; *dropped = hand.dropped;
  if (hand.st != LL_OK || hand.dropped) return hand.st;
  if (hand.nc + hand.ns == 0) { item_prologue(ctx, map, 0, in, out, &st); ctx->last_nc = 0; ctx->last_ns = 0; }   // as register_device reports it
  return st;
}

extern "C" int ll_scan_to_pose(ll_ctx* ctx, const ll_map* map, const void* raw, size_t n, int fmt, int where, double stamp, const ll_pipeline_cfg* pc, const ll_reg_state* in,
                    ll_reg_result* out, int* n_corner_used, int* n_surf_used) {
  if (!ctx || !map || !pc || !in || !out) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  int nc = 0, ns = 0, dropped = 0;
  if (device_handoff(ctx, map, in)) {
    const int st = register_dev_counts(ctx, map, pc, in, out, &nc, &ns, &dropped,
                                       [&] { return scan_front_end_enqueue(ctx, ctx->own_front(), raw, n, fmt, where, stamp, pc); });
    if (st != LL_OK && !(st == LL_ERR_NO_BLOCKS && !dropped)) return st;
    if (n_corner_used) *n_corner_used = nc; if (n_surf_used) *n_surf_used = ns;
    if (dropped) { memset(out, 0, sizeof(*out)); out->status = 1; ctx->set_error("frame dropped: <= 5 petals"); return LL_OK; }
    return st;
  }
  LL_TRY(scan_front_end(ctx, raw, n, fmt, where, stamp, pc, &nc, &ns, &dropped));
  if (n_corner_used) *n_corner_used = nc; if (n_surf_used) *n_surf_used = ns;
  if (dropped) { memset(out, 0, sizeof(*out)); out->status = 1; ctx->set_error("frame dropped: <= 5 petals"); return LL_OK; }
  return register_device(ctx, map, nc, ns, in, out);
}

// Caller-given features where the front end leaves them (tmp_a / tmp_b, counts[5] / [7]), then ll_scan_to_pose's registration on the device
// counts for a whole frame.  n_corner + n_surf > max_features reaches the hand-over kernel's rule, as a front end's counts would.
extern "C" int ll_register_dev_counts(ll_ctx* ctx, const ll_map* map, const void* scan_corner, size_t n_corner, const void* scan_surf, size_t n_surf, int fmt,
                                      int where, const ll_reg_state* in, ll_reg_result* out) {
  if (!ctx || !map || !in || !out || (!scan_corner && n_corner) || (!scan_surf && n_surf)) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  if (!device_handoff(ctx, map, in)) { ctx->set_error("ll_scan_to_pose would register on host-sized counts here"); return LL_ERR_INVALID; }
  if (n_corner > (size_t)ctx->cfg.max_scan_points || n_surf > (size_t)ctx->cfg.max_scan_points) {
    ctx->set_error("more corner or surface features than max_scan_points"); return LL_ERR_CAPACITY;
  }
  static const ll_pipeline_cfg whole = {1, 0, 0.f, 0.f, 0.f, 0.f, 1};   // (only whole_frame is read: no piece is dropped)
  cudaStream_t s = ctx->stream;
  const RegArrays& A = ctx->A;
  const int cnt[2] = {(int)n_corner, (int)n_surf};
  int nc = 0, ns = 0, dropped = 0;
  return register_dev_counts(ctx, map, &whole, in, out, &nc, &ns, &dropped, [&]() -> int {
    LL_TRY(upload_cloud(ctx, s, scan_corner, n_corner, fmt, where, A.tmp_a));
    LL_TRY(upload_cloud(ctx, s, scan_surf, n_surf, fmt, where, A.tmp_b));
    LL_CUDA(ctx, cudaMemcpyAsync(A.counts + 5, &cnt[0], sizeof(int), cudaMemcpyHostToDevice, s));
    LL_CUDA(ctx, cudaMemcpyAsync(A.counts + 7, &cnt[1], sizeof(int), cudaMemcpyHostToDevice, s));
    return front_end_counts_d2h(ctx, s);
  });
}

// Multi-head frame (Mid-100: three Mid-40 heads, launch/rosbag_mid100.launch): Laser_feature::laserCloudHandler runs ONE Livox_laser object over
// the heads in turn and sums their per-piece feature clouds before the VoxelGrids (laser_feature_extractor.hpp:303-380); the mapping node then sees
// one merged feature pair (laser_mapping.hpp:1367-1405).  Heads whose frame has <= 5 petals contribute nothing (:287).
extern "C" int ll_frame_to_pose(ll_ctx* ctx, const ll_map* map, int n_heads, const void* const* raws, const size_t* ns, int fmt, int where, const double* stamps,
                     const ll_pipeline_cfg* pc, const ll_reg_state* in, ll_reg_result* out, int* n_corner_used, int* n_surf_used) {
  if (!ctx || !map || !pc || !in || !out || !raws || !ns || !stamps || n_heads < 1 || n_heads > 8) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  cudaStream_t s = ctx->stream;
  size_t total = 0; for (int h = 0; h < n_heads; h++) total += ns[h];
  if ((int)total > ctx->cfg.max_scan_points) { ctx->set_error("frame (all heads) larger than max_scan_points"); return LL_ERR_CAPACITY; }
  const RegArrays& A = ctx->A;
  int acc_c = 0, acc_s = 0;
  int* hc = ctx->pin->fe_counts; const int* hm = ctx->pin->fe_meta;
  for (int h = 0; h < n_heads; h++) {
    LL_TRY(extract_prepare(ctx, s, raws[h], ns[h], fmt, where, stamps[h]));
    LL_TRY(extract_enqueue(ctx, s, ctx->fe_main));
    const float* d_bounds = nullptr;
    if (!pc->whole_frame) { LL_TRY(launch_piece_bounds(ctx, s, pc->pieces, A.bounds)); d_bounds = A.bounds + 2 * pc->use_piece; }
    LL_TRY(launch_get_features(ctx, s, ctx->fe_main, d_bounds, 0.f, 1.f, A.tmp_a + acc_c, A.tmp_b + acc_s, nullptr, A.counts));
    LL_CUDA(ctx, cudaMemcpyAsync(hc, A.counts, 3 * sizeof(int), cudaMemcpyDeviceToHost, s));
    LL_CUDA(ctx, cudaMemcpyAsync(ctx->pin->fe_meta, ctx->ex.d_meta, sizeof(ctx->pin->fe_meta), cudaMemcpyDeviceToHost, s));
    LL_CUDA(ctx, cudaStreamSynchronize(s));
    if (ns[h] >= 5 && (hm[1] > 5 || pc->whole_frame)) { acc_c += hc[0]; acc_s += hc[1]; }   // meta[1] = laserCloudScans.size()
  }
  LL_TRY(voxel_chains(ctx, ctx->own_front(), pc, acc_c, nullptr, acc_s, nullptr));   // counts[4..7]
  LL_CUDA(ctx, cudaMemcpyAsync(hc, A.counts, 8 * sizeof(int), cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  const int nc = hc[5], nsf = hc[7];
  if (n_corner_used) *n_corner_used = nc; if (n_surf_used) *n_surf_used = nsf;
  LL_TRY(features_fit(ctx, nc, nsf));
  LL_TRY(features_hand_over(ctx, s, A.tmp_a, nc, A.tmp_b, nsf));
  return register_device(ctx, map, nc, nsf, in, out);
}

// Laser_feature::laserCloudHandler for a whole frame, every piece at once (laser_feature_extractor.hpp:303-389): each head extracted once and
// compacted once with bounds 0 ... 1 (its corner / surface / full clouds at the head's base in tmp_a / tmp_b / tmp_c), the slices of every
// piece read from that compaction, piece i's slices of all heads gathered into segment i, then the extractor's and the mapping node's
// VoxelGrids as one segmented pass each: the corner chain on fs.corner, the surface chain on fs.main.  The launch count does not depend on the
// number of pieces.
// The device part: the heads already lie one after another in the extractor's raw array (head h at raw + base[h]) and their scan times in
// pin->head_time.  Each head is extracted with the raw array pointed at its slice.
static int frame_front_end_device(ll_ctx* ctx, const FrontStreams& fs, const FrameArena& fa, int n_heads, const size_t* ns, int pieces, const ll_pipeline_cfg* pc) {
  cudaStream_t s = fs.main, s2 = fs.corner;
  const RegArrays& A = ctx->A;
  ExtractState& e = ctx->ex;
  float4* const raw0 = e.raw;
  const int st = [&]() -> int {
    FrameBases B; int base = 0, max_n = 0;
    for (int h = 0; h < n_heads; h++) {
      B.base[h] = base;
      e.raw = raw0 + base; e.n = (int)ns[h];
      LL_CUDA(ctx, cudaMemcpyAsync(e.d_time, &ctx->pin->head_time[h], sizeof(double), cudaMemcpyHostToDevice, s));
      LL_TRY(extract_enqueue(ctx, s, ctx->fe_main));
      LL_TRY(launch_piece_bounds(ctx, s, pieces, A.bounds));
      LL_TRY(launch_get_features(ctx, s, ctx->fe_main, nullptr, 0.f, 1.f, A.tmp_a + base, A.tmp_b + base, A.tmp_c + base, A.counts));
      LL_TRY(launch_piece_slices(ctx, s, ctx->fe_main, A.bounds, pieces, A.tmp_c + base, &fa.dev->head[h]));
      base += (int)ns[h]; max_n = std::max(max_n, (int)ns[h]);
    }
    LL_TRY(launch_gather_pieces(ctx, s, fa.dev, B, n_heads, pieces, max_n, A.tmp_a, A.tmp_b, fa.cls[0], fa.cls[1]));
    const int cap = pieces * base;   // a piece holds at most every point of the frame once
    LL_CUDA(ctx, cudaEventRecord(fs.fork, s));
    LL_CUDA(ctx, cudaStreamWaitEvent(s2, fs.fork, 0));
    LL_TRY(launch_voxel_grid_segments(ctx, s2, *fa.vg[1], fa.cls[0], cap, fa.dev->seg_end[0], pieces, pc->extractor_leaf_corner, fa.mid[0], fa.dev->mid_end[0]));
    LL_TRY(launch_voxel_grid_segments(ctx, s2, *fa.vg[1], fa.mid[0], cap, fa.dev->mid_end[0], pieces, pc->mapping_leaf_corner, fa.cls[0], fa.dev->out.out_end[0]));
    LL_CUDA(ctx, cudaEventRecord(fs.join, s2));
    LL_TRY(launch_voxel_grid_segments(ctx, s, *fa.vg[0], fa.cls[1], cap, fa.dev->seg_end[1], pieces, pc->extractor_leaf_surf, fa.mid[1], fa.dev->mid_end[1]));
    LL_TRY(launch_voxel_grid_segments(ctx, s, *fa.vg[0], fa.mid[1], cap, fa.dev->mid_end[1], pieces, pc->mapping_leaf_surf, fa.cls[1], fa.dev->out.out_end[1]));
    LL_CUDA(ctx, cudaStreamWaitEvent(s, fs.join, 0));
    LL_CUDA(ctx, cudaMemcpyAsync(&ctx->pin->frame, &fa.dev->out, sizeof(FrameOut), cudaMemcpyDeviceToHost, s));
    return LL_OK;
  }();
  e.raw = raw0;
  return st;
}

int frame_front_end(ll_ctx* ctx, const FrontStreams& fs, const FrameArena& fa, int n_heads, const void* const* raws, const size_t* ns, int fmt, int where,
                    const double* stamps, int pieces, const ll_pipeline_cfg* pc) {
  cudaStream_t s = fs.main;
  size_t base = 0;
  for (int h = 0; h < n_heads; h++) {   // the extractor's bookkeeping of every head in turn, and the uploads (outside the graph)
    ctx->pin->head_time[h] = extract_stamp(ctx, ns[h], stamps[h]);
    LL_TRY(upload_cloud(ctx, s, raws[h], ns[h], fmt, where, ctx->ex.raw + base));
    base += ns[h];
  }
  FrontKey key; key.n_heads = n_heads; std::copy(ns, ns + n_heads, key.ns); key.pieces = pieces; key.pc = *pc;
  return front_graph(ctx, *fa.graph, s, key, true, [&] { return frame_front_end_device(ctx, fs, fa, n_heads, ns, pieces, pc); });
}

extern "C" {

// ---------------------------------------------------------------------------------------------- multi-GPU
int ll_comm_local_handle(ll_ctx* ctx, unsigned char handle[LL_IPC_HANDLE_BYTES]) {
  if (!ctx) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  const size_t comm_bytes = LL_COMM_X_OFF + (size_t)ctx->cfg.max_features * sizeof(double);
  if (!ctx->comm_local) { LL_CUDA(ctx, cudaMalloc(&ctx->comm_local, comm_bytes)); LL_CUDA(ctx, cudaMemset(ctx->comm_local, 0, comm_bytes)); }
  cudaIpcMemHandle_t h; LL_CUDA(ctx, cudaIpcGetMemHandle(&h, ctx->comm_local));
  static_assert(sizeof(cudaIpcMemHandle_t) <= LL_IPC_HANDLE_BYTES, "ipc handle size");
  memset(handle, 0, LL_IPC_HANDLE_BYTES); memcpy(handle, &h, sizeof(h));
  return LL_OK;
}
int ll_comm_connect(ll_ctx* ctx, int rank, int world, const unsigned char* all) {
  if (!ctx || world < 1 || world > 8 || rank < 0 || rank >= world) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  if (!ctx->comm_local) { ctx->set_error("call ll_comm_local_handle first"); return LL_ERR_INVALID; }
  ctx->rank = rank; ctx->world = world;
  for (int p = 0; p < world; p++) {
    if (p == rank) { ctx->comm_peers[p] = ctx->comm_local; continue; }
    cudaIpcMemHandle_t h; memcpy(&h, all + (size_t)p * LL_IPC_HANDLE_BYTES, sizeof(h));
    LL_CUDA(ctx, cudaIpcOpenMemHandle(&ctx->comm_peers[p], h, cudaIpcMemLazyEnablePeerAccess));
  }
  return LL_OK;
}
}  // extern "C"
