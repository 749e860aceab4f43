// Kernel argument structs and host-side launch prototypes shared between translation units.
#pragma once
#include "common.cuh"

struct TreeView {
  const float4* pts;                    // [n_pad] Hilbert-ordered points, w = original index
  const float4* src;                    // [n_src] the cloud in its original order
  const float4* nodes[LL_MAX_LEVELS];   // node records per level (64 float4 each: 32 child boxes); level 0's children are the 32-point buckets
  int n, n_levels;
  const float* bbox;                    // device: map bounding box (min xyz, max xyz)
};
TreeView make_view(const BucketTree& t);
int build_bucket_tree(ll_ctx* ctx, cudaStream_t s, DevBuf& scratch, const float4* d_src, int n_src, BucketTree* t);
size_t tree_scratch_bytes(int n_src);   // what build_bucket_tree carves from `scratch` and from BucketTree::storage for n_src points
size_t tree_storage_bytes(int n_src);
// Bounding box of the finite points (knn.cu): bbox[0..2] = min, bbox[3..5] = max (ll_f2ord encoding), bbox[6] = their count.
// bbox_init_kernel (one warp) resets it; every bbox_kernel launch after that widens it by one more cloud.
__global__ void bbox_init_kernel(int* bbox);
__global__ void bbox_kernel(const float4* __restrict__ src, int n, int* __restrict__ bbox);

struct RegDevState;
struct KnnBlocksArgs {
  TreeView corner, surf;
  const float4* feat;     // [n_corner + n_surf] scan-frame features (x,y,z,timestamp)
  int n_corner, n_surf;
  const double* pose;     // device: q_curr (w,x,y,z), t_curr
  double max_dis_line, max_dis_plane;
  int icp_line, icp_plane;
  float4* blk_a; double* blk_v;
  int* corner_avail; int* surf_avail; int* n_blocks;   // three consecutive counters in RegDevState, cleared before every launch
  int cap, rng_seed;            // residual-block cap (pre-skip of features at 2 x cap, :232-238, :339-345)
  int* seed_ids;                // [M x 5] neighbour ids of the previous ICP iteration (-1 = none): seeds of the next search
  float* knn_d;                 // optional debug output [M x 5]
  const int* perm;              // spatially sorted feature order (corners then surfaces), or null = caller order
  int rank, world; ShardGrid grid; const int* shard_owner;   // sharded map: a query is processed by the rank that owns its cell
  const RegDevState* st;        // motion deblur reads q_last/t_last, t_incre and the Rodrigues terms from here
  int deblur;
};
int launch_knn_query(ll_ctx* ctx, const BucketTree& t, const float4* d_q, int nq, int* d_idx, float* d_d);
int launch_knn_blocks(ll_ctx* ctx, const KnnBlocksArgs& a);
int launch_query_sort(ll_ctx* ctx, cudaStream_t s, DevBuf& scratch, const KnnBlocksArgs& a, int* d_perm);
size_t query_sort_bytes(int M);

// ---------------------------------------------------------------------------------------------- solver (solve.cu)
#include "lm_state.h"   // FnSample, LmState (the state machine itself: lm_core.cuh, included by solve.cu)

struct RegDevState {
  // pose block, contiguous: q_curr(w,x,y,z) t_curr(3) | q_last(4) t_last(3)
  double pose_curr[7];
  double pose_last[7];
  double x[7];                 // m_para_buffer_incremental: q (x,y,z,w), t
  double q_last_opt[4], t_last_opt[3];   // q_last_optimize / t_last_optimize of the ICP loop
  double bound, huber_a, inliner_dis, inlier_ratio, min_icp_R, min_icp_T;
  double inlier_threshold, angular_diff, t_diff, final_cost, initial_cost;
  int corner_avail, surf_avail, n_blocks, icp_done, icp_iter, num_residual_blocks, status, total_lm_iterations, total_evaluations;
  int n_unique; int if_motion_deblur;
  // residual-block cap: m_maximum_allow_residual_block, the seed of ll_cap_uniform_f, and the number of blocks the kNN kernel of this ICP
  // iteration emitted (n_blocks, next to corner_avail: this rank; n_blocks_all: all ranks, = n_blocks unless the map is sharded)
  int cap, rng_seed, n_blocks_all;
  // motion deblur (N1): time-stamp range of refine_blur, and compute_interpolatation_rodrigue's outputs (:607-620) after every solve #2
  double min_ts, max_ts, interp_theta, interp_hat[9], interp_hat_sq[9];
  long long prof[16];  // [8..12]: fused K10 section: L1 + insert, barrier, select, barrier, drop   // master-CTA cycle counters of the solver: eval, wait, grid reduce, lm_step, publish, #evaluations, staging, epilogue
  LmState lm;
};

// Pinned host staging of the small transfers, one field per transfer.  The rule every field relies on: a field the host writes before an
// async copy is not written again until that copy has completed (every entry point synchronises before it returns; register_device reads
// snap[it & 1] only after the event recorded behind its copy).
struct PinnedStage {
  RegDevState state_in;   // the registration state uploaded by register_device / ll_build_blocks / ll_set_blocks
  RegDevState snap[2];    // state read-backs: ICP iteration `it` into snap[it & 1]; the solver parity hooks use snap[0]
  double x[7];            // x of the solver parity hooks
  double pose[7];         // ll_transform / ll_transform_dev
  double mapper_pose[7];  // the mapper's world-frame transform of the new features
  double extract_time;    // ExtractState::d_time
  int fe_counts[12];      // front end: RegArrays::counts ([0..2] get_features, [4..7] VoxelGrid outputs, [10..11] time-stamp range)
  int fe_meta[3];         // front end: ExtractState::d_meta
  int counts[3];          // count read-backs of the single-call entry points
  float bounds[32];       // ll_piece_bounds
};

// Grid-wide exchange area of the solver kernels (one per context, device memory, zeroed once at creation; see solve.cu):
// one tagged 256-byte row per CTA and parity, the broadcast row of the sharded mode, the K10 histograms / candidate list, the generation base.
#define LL_SYNC_ROWS 160
struct SolveSync {
  double rows[2][LL_SYNC_ROWS][32];   // [parity][cta]: 29 sums, [31] = generation tag (low 32 bits)
  double bcast[2][32];                // world > 1: the all-reduced sums, from CTA 0 to the other CTAs of the rank
  unsigned hist[6][2048]; unsigned list_cnt; unsigned _pad[63];   // K10 radix-select histograms + candidate counter (cleared together by every fused launch)
  double list[64];
  unsigned gen;                       // generation base of the next launch; grows monotonically over the life of the context
};

// What one lm_solve_kernel launch does.
enum SolveMode : int {
  SOLVE_FIRST = 0,      // solve #1, then the L1 norm of every block at the solution (sharded mode)
  SOLVE_SECOND = 1,     // drop the blocks above the inlier threshold, solve #2, compose the pose + ICP termination test (sharded mode)
  SOLVE_PLAIN = 2,      // one plain solve (parity hook)
  SOLVE_EVALUATE = 3,   // evaluate once at st->x, sums to st->lm.H / g / x_cost (parity hook)
  SOLVE_FUSED = 4,      // one whole ICP iteration in one launch: solve #1 -> K10 inlier threshold -> solve #2 -> pose
};
struct SolveArgs {
  RegDevState* st;
  SolveSync* sync;
  const float4* feat;        // [M] scan-frame points
  const float4* blk_a;       // [M] (a.xyz, type)
  const double* blk_v;       // [M*3]
  double* l1;                // [M] loss-corrected L1 norm per slot (+inf for invalid slots)
  const double* k10_value;   // SOLVE_SECOND: the K10 order statistic and distinct count (launch_k10_select) for the threshold of solve #2
  const int* k10_n_distinct;
  int M;
  int max_iterations;
  SolveMode mode;
  // multi-GPU
  int rank, world; double* comm_local; double* comm_peer[8];
  // SOLVE_FUSED: solve #1's iteration count and the hash set of the L1 norms (K10)
  int prerun_iterations; unsigned long long* table; unsigned table_mask;
  int cap_check;             // 1: the block count can exceed the cap (host: slots > cap): apply the drop rule (:434-458) while staging
  int deblur;                // 1: *_mb functors (ceres_icp.hpp:81-233), s per block from the feature's time stamp
};
// Layout of the IPC-exported staging buffer of a rank (ll_comm_local_handle):
//   [0, 8192)            2 parities x 8 ranks x 64 doubles: the 29 sums of one evaluation + a generation flag at double index 32
//   [8192, 8192+1024)    control words ([3] count-exchange generation (local), [64..80) 2 parities x 8 block counts written by the peers,
//                        [80..88) count-exchange flags written by the peers): [0] comm_gen (local, monotonic over the life of the context: never reset, so a stale flag can never
//                        match), [1] exchange generation (local), [2] block counter (local), [16..24) exchange flags written by the peers
//   [16384, ...)         L1 exchange buffer X: one double per residual-block slot (max_features)
#define LL_COMM_CTRL_OFF 8192
#define LL_COMM_X_OFF 16384
int launch_solve(ll_ctx* ctx, const SolveArgs& a);
// LL_OK when M residual-block slots fit the shared memory of the solver's CTAs (deblur: the *_mb slot layout), else LL_ERR_CAPACITY with the
// context's error set.  The one copy of the rule launch_solve applies: callers check with it before they enqueue anything.
int solve_capacity(ll_ctx* ctx, int M, int deblur);
int solve_prepare(ll_ctx* ctx);   // once per context: opt the solver kernels in to their dynamic shared memory
// The fused solver's K10 (grid-wide de-duplication + radix select) over n values, +inf / NaN skipped; *d_value, *d_n_distinct on the device.
// The sharded mode's select over the exchanged L1 norms, and the parity hook ll_inlier_select.
int launch_k10_select(ll_ctx* ctx, const double* d_l1, int n, const double* d_ratio, unsigned long long* table, unsigned table_mask, double* d_value, int* d_n_distinct);
// Slots of the hash set of M L1 norms (K10): a power of two >= 2 M.
inline unsigned l1_set_capacity(int M) { unsigned cap = 1024; while (cap < (unsigned)(2 * M)) cap <<= 1; return cap; }
// The hash set's place at the start of a scratch arena.
inline unsigned long long* l1_set_layout(Carve& c, int M) { return c.take<unsigned long long>(l1_set_capacity(M)); }
// Sharded mode, K10: every rank pushes the loss-corrected L1 norms of the slots it owns into every peer's X buffer (NVLink stores), then a
// flag barrier; afterwards X is identical on all ranks (NaN where nobody produced a block).
int launch_l1_exchange(ll_ctx* ctx, const double* d_l1, int M);
// Sharded mode, residual-block cap: all ranks' block counts of this ICP iteration summed into RegDevState::n_blocks_all (peer stores + flags).
int launch_count_exchange(ll_ctx* ctx);

// ---------------------------------------------------------------------------------------------- clouds (cloud.cu)
int upload_cloud(ll_ctx* ctx, const void* src, size_t n, int fmt, int where, float4* d_dst);   // async on ctx->stream
int launch_transform(ll_ctx* ctx, cudaStream_t s, const double* d_pose7, const float4* d_in, int n, float4* d_out);
int launch_pack_strided(ll_ctx* ctx, const float4* d_src, int n, unsigned char* d_dst);   // 16-byte points -> PointCloud2 records (ctx->layout)
// VoxelGrid on device: d_in [n] -> d_out [<= n], *d_n_out on device. n given by host, or by device count d_n_in (may be null).
int launch_voxel_grid(ll_ctx* ctx, cudaStream_t s, DevBuf& scratch, const float4* d_in, int n_cap, const int* d_n_in, float leaf, float4* d_out, int* d_n_out);
size_t voxel_grid_bytes(int n_cap);   // what launch_voxel_grid carves from `scratch`

// ---------------------------------------------------------------------------------------------- extractor (extract.cu)
int extract_alloc(ll_ctx* ctx);   // ExtractState arrays for max_scan_points (ll_ctx_create)
int launch_extract_points(ll_ctx* ctx, int n);   // current_time is read from ctx->ex.d_time
int launch_extract_petals(ll_ctx* ctx, int n, cudaStream_t s, DevBuf& scratch);
int launch_get_features(ll_ctx* ctx, cudaStream_t s, DevBuf& scratch, const float* d_bounds /*min_blur,max_blur on device*/, float min_blur, float max_blur,
                        float4* d_corners, float4* d_surf, float4* d_full, int* d_counts /*3*/);
int launch_piece_bounds(ll_ctx* ctx, int pieces, float* d_start_end /* 2*pieces */);
size_t petals_bytes(int n);         // what launch_extract_petals carves from `scratch`
size_t get_features_bytes(int n);   // what launch_get_features carves from `scratch`

// ---------------------------------------------------------------------------------------------- host driver pieces (api.cu)
int register_device(ll_ctx* ctx, const ll_map* map, int nc, int ns, const ll_reg_state* in, ll_reg_result* out);
int scan_front_end(ll_ctx* ctx, const void* raw, size_t n, int fmt, int where, double stamp, const ll_pipeline_cfg* pc, int* nc_out, int* ns_out, int* dropped);
