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
// The map side's two halves side by side (the index builds of ll_map_build / _rebuild, the mapper's whole-map and append VoxelGrids):
// half(c, stream, scratch) enqueues class c, the corner half (0) on stream2 with scratch2 first, then the surface half (1) on `s` with scratch.
// Both halves are enqueued and the join is always recorded, so `s` is behind both whatever they return; returns the first non-OK status.
template <class F> int map_side_pair(ll_ctx* ctx, cudaStream_t s, F&& half) {
  LL_CUDA(ctx, cudaEventRecord(ctx->sev.fork, s));
  LL_CUDA(ctx, cudaStreamWaitEvent(ctx->stream2, ctx->sev.fork, 0));
  const int st0 = half(0, ctx->stream2, ctx->scratch2);
  const int st1 = half(1, s, ctx->scratch);
  LL_CUDA(ctx, cudaEventRecord(ctx->sev.join, ctx->stream2));
  LL_CUDA(ctx, cudaStreamWaitEvent(s, ctx->sev.join, 0));
  return st0 != LL_OK ? st0 : st1;
}
// Bounding box of the finite points (knn.cu): bbox[0..2] = min, bbox[3..5] = max (ll_f2ord encoding), bbox[6] = their count.
// bbox_init_kernel (one warp) resets it; every bbox_kernel launch after that widens it by one more cloud.
__global__ void bbox_init_kernel(int* bbox);
__global__ void bbox_kernel(const float4* __restrict__ src, int n, int* __restrict__ bbox);

struct RegDevState;
// One registration of a batch (ll_register_batch; ll_register is the batch of one): its features are slots off ... off + n_corner + n_surf of
// the feature arena, corners first.
struct KnnItem {
  int off, n_corner, n_surf;
  int icp_line, icp_plane;
  int cap, rng_seed;            // residual-block cap (pre-skip of features at 2 x cap, :232-238, :339-345), drawn by the item-local feature index
  double max_dis_line, max_dis_plane;
};
struct KnnBlocksArgs {
  TreeView corner, surf;
  const float4* feat;     // [M] scan-frame features (x,y,z,timestamp), the items one after another
  int M, n_items;
  KnnItem item[LL_MAX_BATCH];   // ascending off
  float4* blk_a; double* blk_v;
  int* seed_ids;                // [M x 5] neighbour ids of the previous ICP iteration (-1 = none): seeds of the next search
  float* knn_d;                 // optional debug output [M x 5]
  const int* perm;              // spatially sorted feature order (per item: corners then surfaces), or null = caller order
  int rank, world; ShardGrid grid; const int* shard_owner;   // sharded map (one item): a query is processed by the rank that owns its cell
  RegDevState* st;              // [n_items]: the pose, the deblur terms, icp_done, and the counters corner_avail / surf_avail / n_blocks
                                // (cleared before every launch)
  int deblur;
  // One item whose counts only the device knows (ll_scan_to_pose): {n_corner, n_surf} of item 0, the front end's counts; M and item 0's
  // counts above are then the capacity the launches are sized for.  Null: the counts above are the item's.
  const int* dev_counts;
};
int launch_knn_query(ll_ctx* ctx, const BucketTree& t, const float4* d_q, int nq, int* d_idx, float* d_d);
int launch_knn_blocks(ll_ctx* ctx, const KnnBlocksArgs& a);
int launch_query_sort(ll_ctx* ctx, cudaStream_t s, DevBuf& scratch, const KnnBlocksArgs& a, int* d_perm);
size_t query_sort_bytes(int M, int n_items);

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
  int icp_max_iterations;      // solve #2 sets icp_done when icp_iter reaches it: a batch item stops at its own limit while others run on
  // motion deblur (N1): time-stamp range of refine_blur, and compute_interpolatation_rodrigue's outputs (:607-620) after every solve #2
  double min_ts, max_ts, interp_theta, interp_hat[9], interp_hat_sq[9];
  long long prof[16];  // [8..12]: fused K10 section: L1 + insert, barrier, select, barrier, drop   // master-CTA cycle counters of the solver: eval, wait, grid reduce, lm_step, publish, #evaluations, staging, epilogue
  LmState lm;
};

// The piecewise frame front end (frame_front_end).  get_features decides range membership per point and the class of a point does not
// depend on the range, so the corner / surface / full clouds of piece i are contiguous slices of the whole-scan compaction (bounds 0 ... 1):
// from the prefix count at the first index inside the piece's bounds to the prefix count past the last one.
#define LL_MAX_PIECES 16
struct FrameSlices {                   // one head: per class (corner, surface, full) and piece, the slice of the head's compaction
  int off[3][LL_MAX_PIECES], len[3][LL_MAX_PIECES];
  int tmax[LL_MAX_PIECES];             // ll_f2ord of the largest time stamp of the full slice (-10000: find_min_max_intensity's start value)
  int live;                            // the head has > 5 petals (laser_feature_extractor.hpp:287); else every slice is empty
};
struct FrameBases { int base[LL_MAX_HEADS]; };   // where each head's compaction starts in the class arrays
struct FrameOut {                      // what the host reads after the front end of a frame
  int out_end[2][LL_MAX_PIECES];       // corner / surface: end of piece i's down-sampled features
  int tmax[LL_MAX_PIECES];             // per piece, over the heads
  int heads_live;
};
struct FrameDev {
  FrameSlices head[LL_MAX_HEADS];
  int seg_end[2][LL_MAX_PIECES], mid_end[2][LL_MAX_PIECES];   // gathered segments / the extractor's VoxelGrid outputs
  FrameOut out;
};

// Pinned host staging of the small transfers, one field per transfer.  The rule every field relies on: a field the host writes before an
// async copy is not written again until that copy has completed (every entry point synchronises before it returns; register_device reads
// snap[it & 1] only after the event recorded behind its copy).
struct PinnedStage {
  RegDevState state_in[LL_MAX_BATCH];   // the registration states uploaded by register_batch / ll_build_blocks / ll_set_blocks (item order)
  RegDevState snap[2][LL_MAX_BATCH];    // state read-backs: ICP iteration `it` of every item into snap[it & 1], written by the fused solver launch itself
                                        // (SolveArgs::snap; copied in the sharded mode); the solver parity hooks use snap[0][0]
  double x[7];            // x of the solver parity hooks
  double pose[7];         // ll_transform / ll_transform_dev
  double mapper_pose[7];  // the mapper's world-frame transform of the new features
  double loop_pose[7];    // loop feedback: the step's pose in the odometry frame (loop closure's transform of the step's full cloud)
  double extract_time;    // ExtractState::d_time
  int fe_counts[12];      // front end: RegArrays::counts ([0..2] get_features, [4..7] VoxelGrid outputs, [10..11] time-stamp range)
  int fe_meta[3];         // front end: ExtractState::d_meta
  int counts[3];          // count read-backs of the single-call entry points
  float bounds[32];       // ll_piece_bounds
  double head_time[LL_MAX_HEADS];   // ExtractState::d_time of each head of a piecewise frame (its heads are enqueued without a synchronisation)
  FrameOut frame;         // piecewise frame front end: FrameDev::out
};

// Grid-wide exchange area of the solver kernels (one per context, device memory, zeroed once at creation; see solve.cu):
// one tagged 256-byte row per CTA and parity, the broadcast row of the sharded mode, per CTA group (batch item) the K10 histograms / candidate
// list, the generation base.
#define LL_SYNC_ROWS 160
struct K10Area {
  unsigned hist[6][2048]; unsigned list_cnt; unsigned _pad[63];   // K10 radix-select histograms + candidate counter (cleared together by every fused launch)
  double list[64];
};
struct SolveSync {
  double rows[2][LL_SYNC_ROWS][32];   // [parity][cta]: 29 sums, [31] = generation tag (low 32 bits)
  double bcast[2][32];                // world > 1: the all-reduced sums, from CTA 0 to the other CTAs of the rank
  K10Area k10[LL_MAX_BATCH];          // [group]
  unsigned gen;                       // generation base of the next launch; grows monotonically over the life of the context
  unsigned gen_max, exits;            // launches of several groups: the largest generation any group reached, and the CTAs that have ended
};

// What one lm_solve_kernel launch does.
enum SolveMode : int {
  SOLVE_FIRST = 0,      // solve #1, then the L1 norm of every block at the solution (sharded mode)
  SOLVE_SECOND = 1,     // drop the blocks above the inlier threshold, solve #2, compose the pose + ICP termination test (sharded mode)
  SOLVE_PLAIN = 2,      // one plain solve (parity hook)
  SOLVE_EVALUATE = 3,   // evaluate once at st->x, sums to st->lm.H / g / x_cost (parity hook)
  SOLVE_FUSED = 4,      // one whole ICP iteration in one launch: solve #1 -> K10 inlier threshold -> solve #2 -> pose
};
// One item of a solver launch: its slots, its solve, and (filled in by launch_solve) the CTA group that runs it.
struct SolveItem {
  int off, M;                // slots off ... off + M of the arrays below
  int max_iterations;
  int prerun_iterations;     // SOLVE_FUSED: solve #1's iteration count
  int cap_check;             // 1: the block count can exceed the cap (host: slots > cap): apply the drop rule (:434-458) while staging
  unsigned long long* table; unsigned table_mask;   // SOLVE_FUSED: the hash set of the item's L1 norms (K10)
  int first, n_cta, tile, tiles_per_cta;            // CTAs first ... first + n_cta - 1; `tile` slots per CTA and pass (batch_grid)
};
struct SolveArgs {
  RegDevState* st;           // [n_items]
  SolveSync* sync;
  const float4* feat;        // [slots] scan-frame points
  const float4* blk_a;       // [slots] (a.xyz, type)
  const double* blk_v;       // [slots*3]
  double* l1;                // [slots] loss-corrected L1 norm per slot (+inf for invalid slots)
  const double* k10_value;   // SOLVE_SECOND: the K10 order statistic and distinct count (launch_k10_select) for the threshold of solve #2
  const int* k10_n_distinct;
  SolveMode mode;
  // multi-GPU (one item)
  int rank, world; double* comm_local; double* comm_peer[8];
  int deblur;                // 1: *_mb functors (ceres_icp.hpp:81-233), s per block from the feature's time stamp
  int n_items;               // 1 ... LL_MAX_BATCH; more than one only in SOLVE_FUSED
  SolveItem item[LL_MAX_BATCH];
  // SOLVE_FUSED of one item whose slot count only the device knows (KnnBlocksArgs::dev_counts): M = dev_counts[0] + dev_counts[1]; the launch
  // is sized for item 0's M as a capacity, and the kernel derives the CTA split, cap_check and the hash set's mask from the device M.
  const int* dev_counts;
  // SOLVE_FUSED of an ICP loop (register_batch): pinned host memory [n_items] that each item's master CTA fills with the item's state at the end
  // of the launch (the iteration's snapshot, without a copy of its own), then it clears the item's kNN counters corner_avail / surf_avail /
  // n_blocks for the next iteration's kNN launch.  Null: neither.
  RegDevState* snap;
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
// LL_OK when the residual-block slots M[0 .. n) of a launch's items fit the shared memory of their CTA groups (deblur: the *_mb slot layout),
// else LL_ERR_CAPACITY with the context's error set and *bad_item (may be null) = the first item that does not fit.  The one copy of the rule
// launch_solve applies: callers check with it before they enqueue anything.
int solve_capacity(ll_ctx* ctx, int n, const int* M, int deblur, int* bad_item = nullptr);
int solve_prepare(ll_ctx* ctx);   // once per context: opt the solver kernels in to their dynamic shared memory
// The fused solver's K10 (grid-wide de-duplication + radix select) over n values, +inf / NaN skipped; *d_value, *d_n_distinct on the device.
// The sharded mode's select over the exchanged L1 norms, and the parity hook ll_inlier_select.
int launch_k10_select(ll_ctx* ctx, const double* d_l1, int n, const double* d_ratio, unsigned long long* table, unsigned table_mask, double* d_value, int* d_n_distinct);
// Slots of the hash set of M L1 norms (K10): a power of two >= 2 M.
__host__ __device__ inline unsigned l1_set_capacity(int M) { unsigned cap = 1024; while (cap < (unsigned)(2 * M)) cap <<= 1; return cap; }
// The hash set's place at the start of a scratch arena.
inline unsigned long long* l1_set_layout(Carve& c, int M) { return c.take<unsigned long long>(l1_set_capacity(M)); }
// Sharded mode, K10: every rank pushes the loss-corrected L1 norms of the slots it owns into every peer's X buffer (NVLink stores), then a
// flag barrier; afterwards X is identical on all ranks (NaN where nobody produced a block).
int launch_l1_exchange(ll_ctx* ctx, const double* d_l1, int M);
// Sharded mode, residual-block cap: all ranks' block counts of this ICP iteration summed into RegDevState::n_blocks_all (peer stores + flags).
int launch_count_exchange(ll_ctx* ctx);

// ---------------------------------------------------------------------------------------------- clouds (cloud.cu)
int upload_cloud(ll_ctx* ctx, cudaStream_t s, const void* src, size_t n, int fmt, int where, float4* d_dst);   // async on s
int launch_transform(ll_ctx* ctx, cudaStream_t s, const double* d_pose7, const float4* d_in, int n, float4* d_out);
int launch_pack_strided(ll_ctx* ctx, const float4* d_src, int n, unsigned char* d_dst);   // 16-byte points -> PointCloud2 records (ctx->layout)
// VoxelGrid on device: d_in [n] -> d_out [<= n], *d_n_out on device. n given by host, or by device count d_n_in (may be null).
int launch_voxel_grid(ll_ctx* ctx, cudaStream_t s, DevBuf& scratch, const float4* d_in, int n_cap, const int* d_n_in, float leaf, float4* d_out, int* d_n_out);
// The same over nseg (1 ... 256) disjoint contiguous segments of d_in, segment s ending at the device index d_end[s] (clamped to n_cap; d_end may be
// null when nseg == 1): each segment filtered as if alone, the outputs one segment after another, d_out_end[s] = the end of segment s's output.
int launch_voxel_grid_segments(ll_ctx* ctx, cudaStream_t s, DevBuf& scratch, const float4* d_in, int n_cap, const int* d_end, int nseg, float leaf, float4* d_out, int* d_out_end);
size_t voxel_grid_bytes(int n_cap, int nseg = 1);   // what launch_voxel_grid(_segments) carves from `scratch`
// A chain of nvg (1 or 2) VoxelGrids, each on the previous one's output: in [n_cap points, or the device count *d_n_in clamped to n_cap]
// -> out[0] (*d_n_out[0]) -> out[1] (*d_n_out[1]).
struct VgChainDev { const float4* in; int n_cap; const int* d_n_in; int nvg; float leaf[2]; float4* out[2]; int* d_n_out[2]; };
struct VgChain { VgChainDev d; DevBuf* scratch; cudaStream_t s; };   // scratch and stream of the CUB pass
// nchains (1 or 2) chains ordered on stream s: one launch, one cluster per chain, when every n_cap is small enough, else each chain's CUB passes
// on its own stream (at most one stream other than s: it forks from s through `fork` and s waits for it through `join`).
int launch_voxel_chains(ll_ctx* ctx, cudaStream_t s, const VgChain* c, int nchains, cudaEvent_t fork, cudaEvent_t join);
int voxel_grid_prepare(ll_ctx* ctx);   // once per context: opt the cluster VoxelGrid kernel in to its shared memory and its 16-CTA clusters

// ---------------------------------------------------------------------------------------------- extractor (extract.cu)
int extract_alloc(ll_ctx* ctx);   // ExtractState arrays for max_scan_points (ll_ctx_create)
int launch_extract_points(ll_ctx* ctx, cudaStream_t s, int n);   // current_time is read from ctx->ex.d_time
int launch_extract_petals(ll_ctx* ctx, int n, cudaStream_t s, DevBuf& scratch);
int launch_get_features(ll_ctx* ctx, cudaStream_t s, DevBuf& scratch, const float* d_bounds /*min_blur,max_blur on device*/, float min_blur, float max_blur,
                        float4* d_corners, float4* d_surf, float4* d_full, int* d_counts /*3*/);
int launch_piece_bounds(ll_ctx* ctx, cudaStream_t s, int pieces, float* d_start_end /* 2*pieces */);
size_t petals_bytes(int n);         // what launch_extract_petals carves from `scratch`
size_t get_features_bytes(int n);   // what launch_get_features carves from `scratch`

// ---------------------------------------------------------------------------------------------- piecewise frame front end (extract.cu)
// After launch_get_features(bounds 0 ... 1, full kept) of one head, on the same stream and scratch: the slices of `pieces` pieces from the
// bounds at d_bounds (launch_piece_bounds), and the time-stamp maximum of each full slice (`full` = the head's full cloud).
int launch_piece_slices(ll_ctx* ctx, cudaStream_t s, DevBuf& scratch, const float* d_bounds, int pieces, const float4* full, FrameSlices* out);
// Piece i's slices of every head, in head order, into segment i of dst_c / dst_s; seg_end, out.tmax and out.heads_live of `dev`.
int launch_gather_pieces(ll_ctx* ctx, cudaStream_t s, FrameDev* dev, const FrameBases& B, int n_heads, int pieces, int max_head_n,
                         const float4* src_c, const float4* src_s, float4* dst_c, float4* dst_s);

// ---------------------------------------------------------------------------------------------- cell-map checkpoint (cellmap.cu)
// Cells in the table and live points in the store, current_frame_idx and n_out_of_range; the map is only read.
int cm_count(ll_ctx* ctx, ll_cellmap* m, int* n_cells, int* n_live, int* frame_idx, int* n_out_of_range);
// Incarnations kept beside the live points (the loop image): the sorted, distinct (slot << 32 | epoch) ids the open keyframes hold, on the device.
struct CmHeld { const unsigned long long* ids; int n; };
// The points of a map that an export with `held` keeps: the live ones and those of the held incarnations.
int cm_count_kept(ll_ctx* ctx, ll_cellmap* m, const CmHeld& held, int* n_kept);
// The cells in ascending key then the live points in store order, as the image's cell section holds them (n_cells ll_image_cell, n_live
// ll_image_cell_point, the counts cm_count gave), copied once to host memory `out`; the map is only read.  With `held` (n_live: cm_count_kept's
// count) the held incarnations' points too, then int32 ordinals (cellmap.cuh, cm_ordinal): each cell's current incarnation, each point's.
int cm_export(ll_ctx* ctx, ll_cellmap* m, int n_cells, int n_live, void* out, const CmHeld* held = nullptr);
// An empty map in the state cm_export recorded (records validated by the caller: keys distinct, cell ranks < n_cells; incarnations: the
// ordinals follow the records and become the epochs).  slot_of_rank (may be NULL): each cell's slot in the new table, host memory.
int cm_import(ll_ctx* ctx, ll_cellmap* m, int frame_idx, int n_out_of_range, const void* in, int n_cells, int n_live, bool incarnations = false,
              int* slot_of_rank = nullptr);
// The n_live live points (the count cm_count gave) in store order, as the map stores them, into the device array dst on the context's stream,
// by the export's live-point selection; the map is only read.
int cm_live_points(ll_ctx* ctx, ll_cellmap* m, int n_live, float4* dst);
// The largest max_cells a cell map takes (LL_ERR_INVALID above): its table of 2^30 slots is the largest whose sizes stay within int.
const int MAX_CELLS = 1 << 29;
int64_t table_capacity(int max_cells);   // the hash-table capacity ll_cellmap_create gives a map of max_cells (any int: computed in int64)

// ---------------------------------------------------------------------------------------------- keyframes in the loop image (keyframe.cu)
int kf_cell_count(const ll_keyframe* kf);
unsigned kf_accumulate_frames(const ll_keyframe* kf);
// An open keyframe's cells as the device holds them (ascending key; ids: slot << 32 | epoch), kf_cell_count entries each, to host memory.
int kf_cell_ids(ll_ctx* ctx, const ll_keyframe* kf, unsigned long long* keys, unsigned long long* ids);
// A new keyframe as an open one over map m: n cells (keys ascending, ids at m's slots and epochs) and its append count.
int kf_restore_open(ll_ctx* ctx, ll_cellmap* m, ll_keyframe* kf, const unsigned long long* keys, const unsigned long long* ids, int n, unsigned accumulate_frames);
// A new keyframe as a closed (analyzed) one with what the search and the alignment read again: its info, its four images (4 x 60 x 60 floats)
// and its line then plane clouds (host memory).  Its cell list, per-cell types and all-points cloud are not kept: nothing reads them again.
int kf_restore_closed(ll_ctx* ctx, ll_cellmap* m, ll_keyframe* kf, const ll_keyframe_info& info, const float* img, const void* cloud);

// ---------------------------------------------------------------------------------------------- relocalization (reloc.cu)
int launch_gather_points(ll_ctx* ctx, cudaStream_t s, const float4* src, const int* idx, int n, float4* dst);   // dst[i] = src[idx[i]]
// The field build ll_reloc_field_build and the streaming mapper's recovery share: a field object without storage, its storage (and the build's
// scratch) allocated for n_vox voxels and max_hyp hypotheses, and a build into it that reuses that storage (release: ll_reloc_field_release).
ll_reloc_field* reloc_field_create(int device);
size_t reloc_field_storage_cap(const ll_reloc_field* f);   // bytes its storage holds
int reloc_field_reserve(ll_ctx* ctx, ll_reloc_field* f, long long n_vox, int max_hyp);
int reloc_field_build_into(ll_ctx* ctx, const ll_map* map, float res, int trunc, int max_hypotheses, ll_reloc_field* f);
// a (x) b, the Hamilton product of (w, x, y, z) quaternions in fp64, each component summed left to right as written (the fine rotations, the
// recovery's yaw circle).
void quat_mul(const double* a, const double* b, double* o);

// ---------------------------------------------------------------------------------------------- host driver pieces (api.cu)
// Registration of the features already resident in A.feat (corners then surfaces): the batch of one.  Core of ll_register / ll_scan_to_pose.
int register_device(ll_ctx* ctx, const ll_map* map, int nc, int ns, const ll_reg_state* in, ll_reg_result* out);
// The one limit on the features a registration takes: nc corners plus ns surfaces within max_features, else LL_ERR_CAPACITY ("more features
// than max_features").
int features_fit(ll_ctx* ctx, size_t nc, size_t ns);
// A step's features into A.feat on `s`, where the registration reads them: nc corners from `corner`, then ns surfaces from `surf`.
int features_hand_over(ll_ctx* ctx, cudaStream_t s, const float4* corner, int nc, const float4* surf, int ns);
// The per-scan front end in parts: enqueue on `fs` (bookkeeping, upload, the front end replayed as a graph; its counts land in
// ctx->pin->fe_counts / fe_meta), and, once that work has completed, front_end_counts (the time-stamp range, the counts of the features it
// left in tmp_a / tmp_b, the drop rule (<= 5 petals, :287) and, unless dropped, features_fit).  scan_front_end = both on the context's own
// streams with a synchronisation between them, then the features handed over on the context's stream unless the scan is dropped.
int scan_front_end_enqueue(ll_ctx* ctx, const FrontStreams& fs, const void* raw, size_t n, int fmt, int where, double stamp, const ll_pipeline_cfg* pc);
int front_end_counts(ll_ctx* ctx, const ll_pipeline_cfg* pc, int* nc_out, int* ns_out, int* dropped);
int scan_front_end(ll_ctx* ctx, const void* raw, size_t n, int fmt, int where, double stamp, const ll_pipeline_cfg* pc, int* nc_out, int* ns_out, int* dropped);
// The device arrays of a piecewise frame front end (owned by the streaming mapper): gathered segments of cap points per class, the first
// VoxelGrids' outputs, the segmented VoxelGrids' scratch arenas (vg[0] on the context's stream, vg[1] on stream2), and the graph of the
// device part (everything after the uploads, so the format and the caller's pointers do not enter it), one per arena.
struct FrameArena { FrameDev* dev; float4* cls[2]; float4* mid[2]; int cap; DevBuf* vg[2]; FrontGraph* graph; };
// Every head through the extractor, the slices of every piece, the gathers and the four segmented VoxelGrids (laser_feature_extractor.hpp:
// 303-380, laser_mapping.hpp:1367-1373), enqueued on `fs` without a host synchronisation (the device part replayed as fa.graph once the
// shape repeats); dev->out lands in ctx->pin->frame.  Piece i's features
// are then cls[0] / cls[1] [out_end[.][i - 1], out_end[.][i]).
int frame_front_end(ll_ctx* ctx, const FrontStreams& fs, const FrameArena& fa, int n_heads, const void* const* raws, const size_t* ns, int fmt, int where, const double* stamps,
                    int pieces, const ll_pipeline_cfg* pc);

// ---------------------------------------------------------------------------------------------- spinning-lidar sweeps (spin.cu)
// The streaming mapper's front end of a sweep (ll_mapper_process_sweep(s)): enqueue runs ll_spin_extract's front end on `fs` plus the mapping
// node's input VoxelGrids (pc->mapping_leaf_corner / _surf) and max_t, without a host synchronisation; once that work has completed, finish
// reads the counts (the handle's clouds are then this sweep's of n points): the sweep's features, where they lie, and max_t.
ll_ctx* spin_ctx(const ll_spin* h);
size_t spin_max_points(const ll_spin* h);
int spin_sweep_enqueue(ll_spin* h, const FrontStreams& fs, const void* raw, size_t n, int fmt, int where, const ll_pipeline_cfg* pc);
void spin_sweep_finish(ll_spin* h, size_t n, const float4** corner, int* nc, const float4** surf, int* ns, float* max_t);
const float4* spin_full_cloud(const ll_spin* h, int* n, const int** d_n);   // the last finished sweep's full cloud and its device count
void spin_forget(ll_spin* h);   // the device clouds no longer match the counts (a sweep enqueued ahead of a failed step): nothing extracted

// ---------------------------------------------------------------------------------------------- streaming mapper (mapper.cu, loop.cu)
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
  void clear() { segs.clear(); tail = 0; }
  void release() { buf[0].release(); buf[1].release(); segs.clear(); tail = 0; }
};

// ll_keyframes_repose on device inputs (posegraph.cu).
int keyframes_repose_dev(ll_ctx* ctx, const float4* d_in, int n, const int* seg_end, int n_kf, const ll_pose* poses_ori, const ll_pose* poses_opt, float leaf,
                         float4* d_mid, float4* d_out, int* d_end, int* d_oend, float* d_aff, int* out_end);
extern "C" void pg_odometry_edge(const ll_pose* prev, int id_prev, const ll_pose* cur, int id_cur, ll_pg_edge* out);

// The streaming mapper's loop closure (loop.cu; ll_mapper_set_loop_closure).  The step's full cloud is captured into the loop closure's own
// buffer before the next input's front end may overwrite the context's arrays: loop_scan_cloud after the scan's hand-over (the front end's
// full cloud, compacted again from the extractor's state), loop_frame_clouds after a frame's front end (every published piece's full slices of
// every head); loop_select_piece picks piece i's.  loop_step runs at the end of a mapper step that appended its features (d_pose: the
// registration pose on the device; pushed: the feature history took the step).
struct LoopClosure;
// What loop feedback (ll_mapper_set_loop_feedback; DESIGN.md §4.6.2) reads and moves in the mapper: its two history windows, the frame index
// of each window segment (the windows are pushed and popped together: one index per segment of both), its pose, the pose of its last window
// addition and its refresh flag.
struct MapperWindow { HistoryWindow* his[2]; std::vector<int>* frame; double* q; double* t; double* last_q; double* last_t; bool* map_dirty; };
int  loop_set(ll_ctx* ctx, LoopClosure** lc, const ll_loop_closure_cfg* cfg, const ll_mapper_config& mcfg, int pieces);
void loop_release(LoopClosure* lc);
int  loop_scan_cloud(ll_ctx* ctx, LoopClosure* lc, const ll_pipeline_cfg* pc);
int  loop_frame_clouds(ll_ctx* ctx, LoopClosure* lc, const FrameDev* dev, const size_t* ns, int n_heads, int publish);
// A sweep's full ring-ordered cloud (m_laser_cloud_full_res of the remapped Velodyne pipeline): the n points at `full`, a spin handle's buffer,
// with the device count d_n as its one segment.  Runs before the next sweep's front end may overwrite `full`.
int  loop_sweep_cloud(ll_ctx* ctx, LoopClosure* lc, const float4* full, int n, const int* d_n);
size_t loop_step_capacity(const LoopClosure* lc);   // points of the full cloud one step can hand over (max_scan_points: the world-frame buffer, one append)
void loop_select_piece(LoopClosure* lc, int i);
int  loop_step(ll_ctx* ctx, LoopClosure* lc, const double* d_pose, bool pushed, int frame_index, const MapperWindow& mw);
int  loop_read(LoopClosure* lc, ll_loop_event* out, int cap, int* n, int* n_dropped);
// The loop image (ll_mapper_loop_save / _load / ll_loop_image_info; format: include/loamlivox_b200.h).  stamp: the mapper's binding stamp (the
// fields of ll_loop_image_scalars before `closed`).  loop_load validates everything on the host first, builds a new loop closure and replaces
// *lc only when the whole restore succeeded.
// With loop feedback on, the image (version 3) holds the window's frame indices, and its load sets them in the mapper.
int  loop_save(ll_ctx* ctx, const LoopClosure* lc, const ll_loop_image_scalars& stamp, const MapperWindow& mw, void* image, size_t cap, size_t* bytes);
int  loop_load(ll_ctx* ctx, LoopClosure** lc, const void* image, size_t bytes, const ll_loop_closure_cfg* cfg, const ll_loop_image_scalars& stamp,
               const ll_mapper_config& mcfg, int pieces, const MapperWindow& mw);
int  loop_image_info(const void* image, size_t bytes, ll_loop_image_summary* info);
int  loop_result(const LoopClosure* lc, int* n, int* closed, ll_pose* poses_ori, ll_pose* poses_opt, int cap, ll_pg_edge* edge);
int  loop_cloud(ll_ctx* ctx, const LoopClosure* lc, int k, ll_point* out_host, size_t cap, size_t* n_out, const ll_point** out_dev);
// ll_mapper_set_loop_policy (lc NULL: loop closure off, refused) and ll_mapper_loop_edges
int  loop_set_policy(ll_ctx* ctx, LoopClosure* lc, const ll_loop_policy* p);
int  loop_edges(const LoopClosure* lc, ll_pg_edge* edges, int cap, int* n_loops);
// ll_mapper_set_loop_feedback (lc NULL: loop closure off, refused) and ll_mapper_loop_correction_read
int  loop_set_feedback(ll_ctx* ctx, LoopClosure* lc, const ll_mapper_config& mcfg, int on);
void loop_correction(const LoopClosure* lc, double q_wxyz[4], double t[3], int* n_applied);

// A log of the last entries (recovery's steps, loop closure's events), oldest first: a push into a full log overwrites the oldest unread entry
// and counts it as dropped; a read takes the oldest entries and clears the dropped count.
template <typename T> struct EventLog {
  std::vector<T> ring; size_t first = 0, count = 0; int dropped = 0;   // count entries from ring[first]
  void open(size_t cap) { if (ring.empty()) ring.resize(cap); }
  T* push() {   // the new entry, zeroed
    if (count == ring.size()) { first = (first + 1) % ring.size(); count--; dropped++; }
    T* e = &ring[(first + count) % ring.size()]; count++;
    memset(e, 0, sizeof(*e));
    return e;
  }
  const T& at(size_t k) const { return ring[(first + k) % ring.size()]; }   // the k-th oldest
  void read(T* out, int cap, int* n, int* n_dropped) {
    const size_t k = count < (size_t)cap ? count : (size_t)cap;
    for (size_t i = 0; i < k; i++) out[i] = at(i);
    if (k > 0) { first = (first + k) % ring.size(); count -= k; }
    *n = (int)k;
    if (n_dropped) *n_dropped = dropped;
    dropped = 0;
  }
  void restore(const void* entries, size_t n, int n_dropped) { memcpy(ring.data(), entries, n * sizeof(T)); first = 0; count = n; dropped = n_dropped; }
};

// ---------------------------------------------------------------------------------------------- byte images (checkpoint.cu)
// What the mapper image and the loop image share (format: include/loamlivox_b200.h).  The checks run on the host before anything touches the
// device and give NULL or what is wrong (LL_ERR_INVALID); the writes copy device data on the context's stream, for the caller to synchronise.
template <typename T> T img_get(const uint8_t* p) { T v; memcpy(&v, p, sizeof(T)); return v; }   // unaligned typed read / write
template <typename T> void img_put(uint8_t* p, const T& v) { memcpy(p, &v, sizeof(T)); }
const size_t HIS_HEAD = 16, CELLS_HEAD = 24;   // the fixed part of a history and a cell-map section
// A header of magic[8], uint32 version, uint32 config_bytes, uint64 total_bytes and `sections` (offset, length) pairs.  image_header writes
// it for sections of lengths len[] back to back in index order and returns the image's size; image_structure checks it (magic, a version in
// version ... max_version, the config's size, total_bytes = the image's size, every section inside the image after the header, no two
// overlapping) and gives the sections.  From version more_from on (0: never) the header holds one section more than `sections`.
struct ImageKind {
  const char* magic; const char* name; uint32_t version, max_version; uint32_t config_bytes; const char* config_name; int sections; uint32_t more_from = 0;
  int count(uint32_t v) const { return sections + (more_from && v >= more_from ? 1 : 0); }
};
size_t image_header(const ImageKind& kind, uint32_t version, const uint64_t* len, void* header);
int image_structure(const void* image, size_t bytes, const ImageKind& kind, ll_image_section* sec, std::string* err);
bool finite_xyz(const uint8_t* p);       // the first three floats at p are finite
bool finite_d(const double* d, int n);
// The history section.  The restore pushes segment by segment from one upload and synchronises.  `finite`: every point must be finite (the
// feature histories; the loop closure's full history holds the steps' full clouds as they came).
struct HistoryView { int64_t n_seg = 0, n_pts = 0; const uint8_t* sizes = nullptr; const uint8_t* pts = nullptr; };
uint64_t history_bytes(const HistoryWindow& w);
int history_write(ll_ctx* ctx, const HistoryWindow& w, uint8_t* p);
const char* history_section(const uint8_t* p, uint64_t L, bool finite, HistoryView* v);
int history_restore(ll_ctx* ctx, HistoryWindow& w, const HistoryView& v);
// The cell-map section: cm_count's head and cm_export's records, with incarnations (the loop image) their ordinals too.
struct CellsView {
  int32_t frame_idx = 0, n_oor = 0; int64_t n_cells = 0, n_pts = 0; const uint8_t* rec = nullptr;
  const uint8_t* cur = nullptr; int32_t max_cur = 0; int64_t replaced = 0;   // incarnations: the cells' current ordinals, their largest, points not current
};
uint64_t cells_bytes(const CellsView& n, bool incarnations);
int cells_write(ll_ctx* ctx, ll_cellmap* m, const CellsView& n, uint8_t* p, const CmHeld* held = nullptr);
const char* cells_section(const uint8_t* p, uint64_t L, bool incarnations, CellsView* v);
int cells_restore(ll_ctx* ctx, ll_cellmap* m, const CellsView& v, bool incarnations, int* slot_of_rank = nullptr);
// The load's capacity rule (LL_ERR_CAPACITY): the cells at most half the table of *max_cells (NULL: not checked), at most 2^30 cell-map points
// and 2^31 - 1 history points.
const char* load_capacity(const CellsView& c, const HistoryView& h, const int* max_cells);
