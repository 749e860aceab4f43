/* loamlivox_b200.h — C-ABI of the H100-native (sm_90a) scan-to-map registration hot path of hku-mars/loam_livox.
 *
 * Plain C, POD structs, caller-owned memory, opaque handles, int status (0 = OK, <0 = error, never throws).
 * No global state; distinct ll_ctx objects may be used from distinct threads concurrently (one CUDA stream each),
 * which is how the reference calls the path (one Point_cloud_registration per std::async worker,
 * loam_livox/source/laser_mapping.hpp:1348,1737-1742).
 *
 * The reference has no plugin/FFI layer; the boundary is the three C++ call seams SURVEY.md §8(b) lists.
 * Each entry point below names the reference call it replaces.  Quaternions are (w,x,y,z) unless noted.
 */
#ifndef LOAMLIVOX_B200_H
#define LOAMLIVOX_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- point formats -------------------------------------------------------------------------------- */
typedef struct { float x, y, z, intensity; } ll_point;                   /* 16 B, the device format     */
typedef struct { float x, y, z, _pad0, intensity, _pad1, _pad2, _pad3; } ll_pcl_xyzi; /* == pcl::PointXYZI (32 B),
                                               the reference's PointType: loam_livox/include/tools/common.h:9 */
enum { LL_FMT_XYZI16 = 0, LL_FMT_PCL32 = 1, LL_FMT_STRIDED = 2 /* records described by ll_set_point_layout, e.g. a sensor_msgs/PointCloud2 payload */ };
enum { LL_HOST = 0, LL_DEVICE = 1 };           /* where an input pointer lives                           */

/* ---- status codes --------------------------------------------------------------------------------- */
enum {
  LL_OK = 0,
  LL_ERR_INVALID = -1,    /* bad argument                                                              */
  LL_ERR_CUDA = -2,       /* CUDA runtime error (ll_last_error has the text)                           */
  LL_ERR_CAPACITY = -3,   /* input larger than the context was created for                             */
  LL_ERR_NO_BLOCKS = -4,  /* no residual block survived the gates (reference would dereference an empty
                             std::set at point_cloud_registration.hpp:160)                              */
  LL_ERR_CAP_BINDS = -5   /* no longer returned (kept for ABI stability): the residual-block cap (:232-238,:339-345,:434-458) is implemented,
                             see ll_reg_state::rng_seed */
};

/* ---- pt_type / pt_label bit masks (livox_feature_extractor.hpp:82-103) --------------------------- */
enum { LL_PT_NORMAL = 0, LL_PT_000 = 1, LL_PT_TOO_NEAR = 2, LL_PT_REFLECTIVITY_LOW = 4, LL_PT_REFLECTIVITY_HIGH = 8,
       LL_PT_CIRCLE_EDGE = 16, LL_PT_NAN = 32, LL_PT_SMALL_VIEW_ANGLE = 64 };
enum { LL_LABEL_INVALID = -1, LL_LABEL_UNLABELED = 0, LL_LABEL_CORNER = 1, LL_LABEL_SURFACE = 2, LL_LABEL_NEAR_NAN = 4,
       LL_LABEL_NEAR_ZERO = 8 };

typedef struct ll_ctx ll_ctx;
typedef struct ll_map ll_map;

/* Context configuration.  The extractor fields are the ones Laser_feature writes into Livox_laser
 * (laser_feature_extractor.hpp:152-154,854,859); capacities size the device arenas once. */
typedef struct {
  float corner_curvature;     /* feature_extraction/corner_curvature   (YAML 0.1)   */
  float surface_curvature;    /* feature_extraction/surface_curvature  (YAML 0.005) */
  float minimum_view_angle;   /* feature_extraction/minimum_view_angle (YAML 5)     */
  float livox_min_dis;        /* feature_extraction/livox_min_dis      (0.1)        */
  float livox_min_sigma;      /* feature_extraction/livox_min_sigma    (7e-4)       */
  float max_fov_deg;          /* Livox_laser::max_fov (17)                          */
  float time_interval_pts;    /* Livox_laser::m_time_internal_pts (1e-5)            */
  int   max_scan_points;      /* capacity: raw points per scan                      */
  int   max_features;         /* capacity: corner + surface features per registration */
} ll_config;
void ll_config_default(ll_config* cfg);

int  ll_ctx_create(const ll_config* cfg, int device, ll_ctx** out);
void ll_ctx_destroy(ll_ctx* ctx);
/* Optional: run one toy registration now, so that the module loads and the first cooperative launch CUDA defers to first use
 * do not land in the first registered scan.  ll_mapper_create calls it; nothing else depends on it. */
int  ll_ctx_warmup(ll_ctx* ctx);
const char* ll_last_error(const ll_ctx* ctx);
/* CUDA stream of the context as a cudaStream_t cast to void* (all work of a context is enqueued on it, except the front end of the sequence
 * calls ll_mapper_process_frames / _scans / _sweeps, which runs on streams of its own and has completed when they return). */
void* ll_ctx_stream(ll_ctx* ctx);
int  ll_ctx_sync(ll_ctx* ctx);

/* ---- S1: feature extraction ------------------------------------------------------------------------ */
/* Replaces Livox_laser::extract_laser_features (livox_feature_extractor.hpp:722-766; projection_scan_3d_2d
 * :458-607, compute_features :361-455, split_laser_scan :657-719).  `raw` is one sensor frame in scan order.
 * *n_scans receives laserCloudScans.size() (the caller drops the frame when it is <= 5,
 * laser_feature_extractor.hpp:287).  Per-scan state stays on the device for ll_get_features. */
int ll_extract(ll_ctx* ctx, const void* raw, size_t n, int fmt, int where, double stamp, int* n_scans);
/* Forget the cross-scan state of the extractor (m_first_receive_time, m_last_maximum_time_stamp): a fresh Livox_laser object. */
int ll_extract_reset(ll_ctx* ctx);
/* Piece bounds of laser_feature_extractor.hpp:313-323 (fraction of the frame covered by each piece). */
int ll_piece_bounds(ll_ctx* ctx, int pieces, float* start, float* end);
/* Replaces Livox_laser::get_features (livox_feature_extractor.hpp:219-272).  Host outputs, each sized n. */
int ll_get_features(ll_ctx* ctx, float minimum_blur, float maximum_blur, ll_point* corners, size_t* n_corners,
                    ll_point* surface, size_t* n_surface, ll_point* full, size_t* n_full);
/* Debug/parity view of the per-point state (Pt_infos, livox_feature_extractor.hpp:118-133); any pointer may be NULL. */
int ll_extract_point_info(ll_ctx* ctx, int32_t* pt_type, int32_t* pt_label, float* curvature, float* view_angle,
                          float* depth_sq2, float* time_stamp, float* polar_dis_sq2, int32_t* polar_direction);
int ll_extract_split_idx(ll_ctx* ctx, int32_t* out, int cap, int* n_out);
/* Parity view of the petal angle (scan_id_index, livox_feature_extractor.hpp:591-597) of each segment between consecutive split
 * indices: *n_out = n_split - 1 when the scan has at least 6 split indices, else 0.  Up to cap values are written. */
int ll_extract_petal_angles(ll_ctx* ctx, float* out, int cap, int* n_out);

/* ---- a5: voxel-grid down-sampling ------------------------------------------------------------------ */
/* Replaces pcl::VoxelGrid<PointXYZI>::filter at laser_feature_extractor.hpp:372-380 and
 * laser_mapping.hpp:491,509,533-537,1367-1373,1434-1437.  `out` must hold n points. */
int ll_voxel_downsample(ll_ctx* ctx, const void* in, size_t n, int fmt, int where, float leaf, ll_point* out, size_t* n_out);
/* The same over n_seg (1 ... 256) disjoint contiguous segments of one host cloud, in one device pass: segment k is [seg_end[k - 1], seg_end[k])
 * (seg_end ascending, <= n; points past the last end belong to no segment).  Each segment is filtered exactly as ll_voxel_downsample filters it
 * alone (own bounds, grid and int32-overflow pass-through; equal voxels of two segments never merge).  out receives the segments' outputs one
 * after another (at most n points), n_out_per_seg[k] their counts.  What the streaming mapper's piecewise front end runs (ll_mapper_process_frame). */
int ll_voxel_downsample_segments(ll_ctx* ctx, const ll_point* in, size_t n, const size_t* seg_end, int n_seg, float leaf, ll_point* out, size_t* n_out_per_seg);

/* ---- S2: map snapshot + index ---------------------------------------------------------------------- */
/* Replaces pcl::KdTreeFLANN::setInputCloud x2 in Laser_mapping::update_buff_for_matching
 * (laser_mapping.hpp:544-545) and in the 4-argument registration overload (point_cloud_registration.hpp:596-597).
 * The two world-frame clouds are copied to HBM and indexed; the handle is immutable and may be shared. */
int  ll_map_build(ll_ctx* ctx, const void* corner, size_t n_corner, const void* surf, size_t n_surf, int fmt, int where, ll_map** out);
/* Re-index an existing snapshot in place, reusing its device buffers (the per-scan refresh, laser_mapping.hpp:533-545). Not concurrent with searches of `map`. */
int  ll_map_rebuild(ll_ctx* ctx, ll_map* map, const void* corner, size_t nc, const void* surf, size_t ns, int fmt, int where);
void ll_map_release(ll_map* map);
size_t ll_map_size(const ll_map* map, int which /*0 corner, 1 surface*/);
/* Multi-GPU (config C4): every rank is given the same two clouds and keeps (copies to HBM and indexes) only its shard: the points of the cells
 * it owns plus every point within halo_corner / halo_surf metres of one of those cells.  Cells are cubes of cell_size metres on a grid over the
 * bounding box of the whole map; in Morton order they are cut into `world` contiguous ranges of (nearly) equal point count, rank r owns range r;
 * border cells extend outwards without bound.  With halo >= sqrt(maximum_dis_line_for_match) (1.42 m) and sqrt(maximum_dis_plane_for_match)
 * (7.07 m) -- the squared-distance gates of point_cloud_registration.hpp:64-65,254,353 -- every accepted correspondence has exactly the neighbours
 * a search of the whole map finds (ll_register refuses gates wider than the halo).  ll_register on a sharded map emits residual blocks only for the
 * features whose cell (at the current pose) this rank owns and all-reduces the normal equations inside the solver kernel (ll_comm_*).
 * Indices returned by ll_knn on a sharded map refer to the shard's own compacted clouds. */
int  ll_map_build_sharded(ll_ctx* ctx, const void* corner, size_t n_corner, const void* surf, size_t n_surf, int fmt, int where,
                          int rank, int world, float cell_size, float halo_corner, float halo_surf, ll_map** out);
typedef struct { int rank, world; float cell_size, halo_corner, halo_surf; float origin[3]; int dims[3]; long long kept_corner, kept_surf, total_corner, total_surf; } ll_shard_info;
/* Grid, halo and shard sizes of a map; owner_out (dims[0]*dims[1]*dims[2] ints, x fastest; may be NULL) receives the rank owning every cell. */
int  ll_map_shard_info(const ll_map* map, ll_shard_info* info, int* owner_out, size_t owner_cap);
/* The partition rule alone (pure host code): points per cell in, owner per cell out. */
int  ll_shard_plan(const int* cell_counts, const int dims[3], int world, int* owner_out);

/* Parity hook for pcl::KdTreeFLANN::nearestKSearch(k = 5) (point_cloud_registration.hpp:249,351): world-frame
 * queries in, 5 indices (into the cloud given to ll_map_build, -1 when fewer exist) and float squared distances out. */
int ll_knn(ll_ctx* ctx, const ll_map* map, int which, const ll_point* queries, size_t nq, int32_t* idx5, float* sqdist5);

/* ---- S3: registration ------------------------------------------------------------------------------ */
/* Inputs of Point_cloud_registration: exactly what Laser_mapping::init_pointcloud_registration copies
 * (laser_mapping.hpp:1266-1297) plus the members Scene_alignment pokes (scene_alignment.hpp:233-243,292-306). */
typedef struct {
  int    if_motion_deblur;                /* m_if_motion_deblur: *_mb functors + interpolated matching */
  int    current_frame_index;             /* m_current_frame_index                                     */
  int    mapping_init_accumulate_frames;  /* m_mapping_init_accumulate_frames                          */
  int    icp_max_iterations;              /* m_para_icp_max_iterations                                 */
  int    cere_max_iterations;             /* m_para_cere_max_iterations                                */
  int    cere_prerun_times;               /* m_para_cere_prerun_times (2)                              */
  int    icp_plane, icp_line;             /* ICP_PLANE, ICP_LINE                                       */
  int    maximum_allow_residual_block;    /* m_maximum_allow_residual_block: features are pre-skipped when their class has more than 2 x this
                                             (:232-238,:339-345) and blocks dropped with probability 1 - cap/M when M exceed it (:434-458)     */
  int    rng_seed;                        /* seed of the counter-based generator that replaces the reference's std::random_device-seeded
                                             m_rand_float (tools_random.hpp:18-25): same seed, same kept blocks, on any GPU count             */
  double para_max_angular_rate;           /* m_para_max_angular_rate (deg, reject gate)                */
  double para_max_speed;                  /* m_para_max_speed (bound on |t_incre[j]|)                  */
  double max_final_cost;                  /* m_max_final_cost                                          */
  double minimum_pt_time_stamp, maximum_pt_time_stamp;
  double minimum_icp_R_diff, minimum_icp_T_diff;
  double inliner_dis, inlier_ratio;       /* m_inliner_dis (0.02), m_inlier_ratio (0.80)               */
  double maximum_dis_plane_for_match;     /* 50.0, compared with a SQUARED distance (:353)             */
  double maximum_dis_line_for_match;      /* 2.0,  compared with a SQUARED distance (:254)             */
  double huber_a;                         /* ceres::HuberLoss(0.1) (:220)                              */
  double q_w_last[4], t_w_last[3];        /* m_q_w_last, m_t_w_last                                    */
  double q_w_curr[4], t_w_curr[3];        /* m_q_w_curr, m_t_w_curr                                    */
  double para_buffer_incremental[7];      /* m_para_buffer_incremental: q (x,y,z,w) then t             */
} ll_reg_state;
/* performance_precision.yaml + launch/rosbag.launch values, EXCEPT the two knobs SURVEY.md 8(d) raises for the 30k-feature benchmark scans:
 * maximum_allow_residual_block = 1e6 (no random drop) and max_final_cost = 1e9 (the shipped 2.0 assumes <= 200 blocks). */
void ll_reg_state_default(ll_reg_state* s);
/* The shipped values exactly: config/performance_precision.yaml (realtime = 0: cap 200) or performance_realtime.yaml (realtime = 1: cap 150),
 * max_allow_final_cost 2.0, launch/rosbag.launch:9-11 (20 deg, 0.3 m). */
void ll_reg_state_yaml(ll_reg_state* s, int realtime);
/* The uniform float in [0,1) the cap draws for (seed, ICP iteration, stream 0 corner pre-skip / 1 surface pre-skip / 2 drop, index). */
float ll_cap_uniform(int seed, int icp_iteration, int stream, int index);

typedef struct {
  int    status;                 /* return value of find_out_incremental_transfrom: 1 accepted or skipped, 0 rejected */
  int    registered;             /* 1 when the ICP branch ran (:199)                                    */
  int    num_residual_blocks;    /* summary.num_residual_blocks of the last solve                       */
  int    icp_iterations, corner_used, surf_used;
  int    total_lm_iterations, total_evaluations;
  double q_w_curr[4], t_w_curr[3];   /* m_q_w_curr, m_t_w_curr                                          */
  double q_w_incre[4], t_w_incre[3]; /* m_q_w_incre (w,x,y,z), m_t_w_incre                              */
  double inlier_threshold;       /* m_inlier_threshold after the final/initial cost rescale (:559)      */
  double final_cost, initial_cost;
  double angular_diff, t_diff;   /* m_angular_diff (deg), m_t_diff                                      */
  float  gpu_ms_total, gpu_ms_knn;  /* CUDA-event timings of this call; gpu_ms_knn = first kNN launch     */
  float  gpu_ms_knn_all, gpu_ms_solve_all, gpu_ms_select_all, gpu_ms_sort; /* sums over the ICP iterations */
} ll_reg_result;

/* Replaces Point_cloud_registration::find_out_incremental_transfrom (point_cloud_registration.hpp:163-583):
 * ICP outer loop; per iteration pointAssociateToMap + 5-NN of every feature (:230-432), gates, residual blocks,
 * Solve #1 (2 iterations), inlier selection (:476-499), Solve #2, pose composition, termination (:514-531), reject
 * gate (:561-573).  Returns LL_OK and fills `out` (out->status carries the reference's 0/1); <0 on error. */
int ll_register(ll_ctx* ctx, const ll_map* map, const void* scan_corner, size_t n_corner, const void* scan_surf, size_t n_surf,
                int fmt, int where, const ll_reg_state* in, ll_reg_result* out);

/* n independent registrations against one map in one call (several robots in one prior map, the keyframes of a recorded sequence, several
 * initial guesses for one scan): one kNN launch and one solver launch per ICP iteration for all of them, the solver's cooperative grid cut into
 * one CTA group per item.  Item i is (corners[i], n_corner[i], surfs[i], n_surf[i], in[i]); items may point to the same scan.
 * out[i] and item_status[i] are what ll_register(ctx, map, corners[i], ..., &in[i], &out[i]) would return for item i alone -- the :199 gate, the
 * reject gate, the residual-block cap with in[i].rng_seed (drawn by the item-local feature index), in[i].icp_max_iterations -- except that the
 * gpu_ms_* fields of every out[i] time the whole batch.  The pose agrees with the single call to the last bits (the order of the solver's
 * grid reduce follows the CTA count of the item's group, which depends on the batch).
 * item_status[i] = LL_OK, or LL_ERR_NO_BLOCKS when item i would fail alone; such an item drops out and the others carry on.  The call itself
 * returns LL_OK, or, before anything is enqueued (the error text names the item): LL_ERR_INVALID for n outside 1 ... LL_MAX_BATCH, a null
 * pointer, a sharded map or items that disagree on if_motion_deblur; LL_ERR_CAPACITY when the features of all items exceed max_features or the
 * slots of an item do not fit the shared memory of its CTA group. */
#define LL_MAX_BATCH 16
int ll_register_batch(ll_ctx* ctx, const ll_map* map, int n, const void* const* corners, const size_t* n_corner, const void* const* surfs,
                      const size_t* n_surf, int fmt, int where, const ll_reg_state* in, ll_reg_result* out, int* item_status);

/* Step-by-step parity hooks (tests): one ICP iteration's residual blocks at the pose in `in`
 * (type 0 invalid / 1 line / 2 plane, a[3], v[3] per slot; slots = corner features then surface features) ... */
int ll_build_blocks(ll_ctx* ctx, const ll_map* map, const void* scan_corner, size_t n_corner, const void* scan_surf, size_t n_surf,
                    int fmt, int where, const ll_reg_state* in, int32_t* type, double* a3, double* v3, int* corner_avail, int* surf_avail);
/* ... and the loss-corrected normal equations at x (q x,y,z,w ; t): out28 = 21 upper-triangular JtJ (row-major), 6 Jtr, cost. */
int ll_normal_equations(ll_ctx* ctx, const double x[7], double out28[28]);
/* ... and one ceres::Solve-equivalent on the blocks currently resident (max_iterations as in Solver::Options). */
int ll_solve(ll_ctx* ctx, int max_iterations, double x_io[7], double* initial_cost, double* final_cost, int* iterations);
/* ... and compute_inlier_residual_threshold (point_cloud_registration.hpp:153-161) over n caller-given L1 norms (non-negative; n <= max_features).
 * The grid-wide select of the fused solver kernel, the same kernel the sharded mode runs between its two solves.
 * +inf and NaN entries are not residuals.  *n_distinct = number of distinct values; *value = element min(floor(ratio n), n-1) of them
 * (0 when there is none). */
int ll_inlier_select(ll_ctx* ctx, const double* l1, size_t n, double ratio, double* value, int* n_distinct);
/* ... and caller-given residual blocks in place of ll_build_blocks': n slots (n <= max_features and within the solver's shared memory, else
 * LL_ERR_CAPACITY before anything is enqueued), type 0 invalid / 1 line / 2 plane, the feature p (scan frame; intensity = time stamp, the blur
 * factor of the *_mb functors comes from it as in a registration), the anchor a3 (fp32, as the kNN kernel stores it) and the direction / normal
 * v3.  The state `in` is loaded as ll_register loads it (last pose, loss, bounds, inlier rule, if_motion_deblur).  ll_normal_equations, ll_solve
 * and ll_solve_fused then run the unchanged staging and evaluation of the solver kernel over exactly these blocks. */
int ll_set_blocks(ll_ctx* ctx, const ll_reg_state* in, size_t n, const int32_t* type, const ll_point* p, const float* a3, const double* v3);
/* ... and one fused ICP iteration of the solver over the resident blocks (one launch, as ll_register runs it): solve #1 (prerun iterations) from
 * x_io, the loss-corrected L1 norm of every slot, the inlier threshold max(inliner_dis, K10 order statistic), the drop of the blocks above it,
 * solve #2 (max_iterations).  x_io <- solve #2's result; *n_distinct = distinct finite L1 norms, *n_kept = blocks solve #2 evaluated,
 * l1_out[n] (or NULL) = the L1 norms (+inf for invalid slots), iterations[2] = LM iterations of solve #1 and #2. */
int ll_solve_fused(ll_ctx* ctx, int prerun, int max_iterations, double x_io[7], double* threshold, int* n_distinct, int* n_kept, double* l1_out,
                   int iterations[2]);
/* ... and caller-given features through ll_scan_to_pose's registration on the front end's device-side counts (the capacity-sized sort, kNN and
 * solver launches that read the counts on the device), for a whole frame: the features go where the front end leaves them and that same path
 * runs.  Returns and fills `out` as ll_register on the same features would, except: LL_ERR_INVALID when ll_scan_to_pose would take the
 * host-sized path for this context, map and state; LL_ERR_CAPACITY when n_corner or n_surf exceeds max_scan_points (both with nothing
 * enqueued).  n_corner + n_surf > max_features is refused on the device as a front end's counts are: LL_ERR_CAPACITY. */
int ll_register_dev_counts(ll_ctx* ctx, const ll_map* map, const void* scan_corner, size_t n_corner, const void* scan_surf, size_t n_surf,
                           int fmt, int where, const ll_reg_state* in, ll_reg_result* out);

/* ---- N4: loop-closure reuse of S3 ----------------------------------------------------------------------- */
/* Replaces Scene_alignment::find_tranfrom_of_two_mappings (scene_alignment.hpp:269-353) from the point where the four feature clouds exist:
 * three coarse-to-fine registrations (leaf x8, x4, x1; twice the ICP iterations at the finest) of the target keyframe's features against the source
 * keyframe's, ICP_LINE = 0, on one persistent registration object (increment and pose carry over between scales, :233-243,292-306).
 * out = the state after the last scale run (q_w_curr / t_w_curr = the transform of keyframe b into keyframe a; inlier_threshold = the score
 * Scene_alignment returns).  *scales_run <= 3 (stops early when inlier_threshold > 2 x accepted_threshold, :349-350). */
typedef struct {
  float  line_res, plane_res;          /* Scene_alignment::m_line_res / m_plane_res (0.4 / 0.4, :27-28)                                  */
  int    maximum_icp_iteration;        /* m_maximum_icp_iteration (10, :35)                                                              */
  int    maximum_residual_block;       /* m_para_scene_alignments_maximum_residual_block (5000, :34)                                     */
  float  accepted_threshold;           /* m_accepted_threshold (0.2, :36)                                                                */
  int    rng_seed;                     /* see ll_reg_state::rng_seed                                                                      */
  double t_init[3];                    /* keyframe_a->get_center() - keyframe_b->get_center() (:303)                                     */
} ll_align_cfg;
void ll_align_cfg_default(ll_align_cfg* cfg);
int  ll_scene_align(ll_ctx* ctx, const void* source_line, size_t n_sl, const void* source_plane, size_t n_sp, const void* target_line, size_t n_tl,
                    const void* target_plane, size_t n_tp, int fmt, int where, const ll_align_cfg* cfg, ll_reg_result* out, int* scales_run);

/* ---- a7: pointAssociateToMap over a cloud ----------------------------------------------------------- */
/* Replaces Point_cloud_registration::pointcloudAssociateToMap (point_cloud_registration.hpp:673-685, non-deblur
 * branch of :622-661): p_w = q*p + t in fp64, stored as fp32, intensity passed through. */
int ll_transform(ll_ctx* ctx, const double q_wxyz[4], const double t[3], const void* in, size_t n, int fmt, int where, ll_point* out);

/* ---- whole per-scan step (what Laser_feature::laserCloudHandler + Laser_mapping::process_new_scan do) ------ */
typedef struct {
  int   pieces;               /* common/piecewise_number; only piece 0 is registered (odom_mode 0, :385)    */
  int   use_piece;            /* which piece's features to register (0)                                      */
  float extractor_leaf_corner;/* laser_feature_extractor.hpp:193 (line_res)                                  */
  float extractor_leaf_surf;  /* laser_feature_extractor.hpp:192 (plane_res / 2)                             */
  float mapping_leaf_corner;  /* laser_mapping.hpp:1367-1373 (line_res)                                      */
  float mapping_leaf_surf;    /* (plane_res)                                                                 */
  int   whole_frame;          /* 1: ignore pieces, use min_blur = 0, max_blur = 1                            */
} ll_pipeline_cfg;
/* raw scan -> features -> VoxelGrid x2 -> registration against `map`, without leaving the device. */
int ll_scan_to_pose(ll_ctx* ctx, const ll_map* map, const void* raw, size_t n, int fmt, int where, double stamp,
                    const ll_pipeline_cfg* pc, const ll_reg_state* in, ll_reg_result* out, int* n_corner_used, int* n_surf_used);

/* Multi-head frames (Mid-100 = three Mid-40 heads, launch/rosbag_mid100.launch:6): ONE extractor handles the heads in turn and the per-piece feature
 * clouds of the heads are summed before the VoxelGrids (laser_feature_extractor.hpp:303-380, 339-389); then as ll_scan_to_pose.  raws / ns / stamps have n_heads
 * entries (<= 8); the context's max_scan_points must cover the whole frame.  A head whose frame has <= 5 petals contributes nothing (:287). */
int ll_frame_to_pose(ll_ctx* ctx, const ll_map* map, int n_heads, const void* const* raws, const size_t* ns, int fmt, int where, const double* stamps,
                     const ll_pipeline_cfg* pc, const ll_reg_state* in, ll_reg_result* out, int* n_corner_used, int* n_surf_used);

/* ---- a14: device-resident voxel-cell map (matching_mode 1) ---------------------------------------------- */
/* Replaces Points_cloud_map<float> as the matching path uses it (cell_map_keyframe.hpp:476-1000): `resolution` is what
 * Laser_mapping passes to set_resolution (1.0 => 0.5 m cells, :674-679), `revisit_threshold` = m_minimum_revisit_threshold
 * (common/threshold_cell_revisit, >= 1).  max_cells sizes the hash table (0 = 1 Mi cells; at most 2^29, LL_ERR_INVALID above). */
typedef struct ll_cellmap ll_cellmap;
int  ll_cellmap_create(ll_ctx* ctx, float resolution, int revisit_threshold, int max_cells, ll_cellmap** out);
void ll_cellmap_release(ll_cellmap* map);
/* Points_cloud_map::append_cloud (cell_map_keyframe.hpp:619-672; a call while the map has no cell = set_point_cloud :578-617). xyz only.
 * Points with a non-finite coordinate are dropped.  Points whose cell index is outside -2^20 ... 2^20 - 1 on an axis are dropped too, and
 * the append then returns LL_ERR_INVALID after completing with the others.  LL_ERR_CAPACITY when the table is more than half full. */
int  ll_cellmap_append(ll_ctx* ctx, ll_cellmap* map, const void* pts, size_t n, int fmt, int where);
/* update_buff_for_matching, matching_mode 1, for one of the two maps (laser_mapping.hpp:475-516): find_cells_in_radius(t, search_range)
 * (cell_map_keyframe.hpp:761-788) + if_pt_in_fov (laser_mapping.hpp:310-324) + per-cell VoxelGrid(leaf) + optional down-sample-and-replace
 * (m_down_sample_replace).  The concatenated cloud stays on the device (*out_dev, valid until the next call on this map) and is copied to
 * out_host (cap points) when out_host != NULL.  Cells are visited in ascending (k, j, i) index order (the PCL octree order is unspecified).
 * A leaf finer than the cell size / 512 is LL_ERR_INVALID: PCL would pass a cell through unfiltered when its voxel count overflows int32. */
int  ll_cellmap_assemble(ll_ctx* ctx, ll_cellmap* map, const double q_w_curr[4], const double t_w_curr[3], float search_range, float fov_deg, float leaf,
                         int down_sample_replace, ll_point* out_host, size_t cap, size_t* n_out, int* cells_in_fov, const ll_point** out_dev);
/* Allocate now for `store_points` stored points and appends of up to `scan_points`: no allocation afterwards while the store stays below that. */
int  ll_cellmap_reserve(ll_ctx* ctx, ll_cellmap* map, size_t store_points, size_t scan_points);
int  ll_cellmap_stats(ll_ctx* ctx, ll_cellmap* map, int* cells, int* stored_points, int* frame_idx);

/* ---- streaming odometry: Laser_mapping::process_new_scan + update_buff_for_matching (matching_mode 0 and 1) ------------------------- */
typedef struct {
  float line_resolution, plane_resolution;      /* feature_extraction/mapping_{line,plane}_resolution (laser_mapping.hpp:661-662)          */
  float cell_resolution;                        /* m_pt_cell_resolution (1.0 => 0.5 m cells)                                               */
  int   threshold_cell_revisit;                 /* common/threshold_cell_revisit                                                           */
  float maximum_search_range_corner, maximum_search_range_surface, maximum_in_fov_angle;   /* mapping/... (:691-695)                      */
  int   down_sample_replace;                    /* m_down_sample_replace (:277)                                                            */
  int   max_cells;                              /* hash-table sizing of each cell map (0 = 1 Mi cells; at most 2^29)                       */
  int   matching_mode;                          /* mapping/matching_mode (:689): 0 = sliding window of the last maximum_history_size feature clouds
                                                   (:518-531,1439-1478; what both shipped YAMLs select), 1 = cells in range and in the FOV (:471-516)   */
  int   maximum_history_size;                   /* mapping/maximum_histroy_buffer (:687; YAML 400 / 200)                                   */
  int   reserve_map_points;                     /* device memory reserved at creation, per feature kind, for the match map (history window / assembled
                                                   cells, its VoxelGrid, snapshot and index): nothing is reallocated while the map stays below it
                                                   (default 4 Mi points >= maximum_history_size x down-sampled features per scan; 0 = grow on
                                                   demand, by doubling)                                                                     */
  int   reserve_store_points;                   /* same for each cell map's point store (default 4 Mi points; the store of mode 0 only ever grows) */
  ll_pipeline_cfg pipeline;                     /* feature-extraction glue (leaves, pieces)                                                */
  ll_reg_state reg;                             /* registration parameters; the poses in it are the initial pose                           */
} ll_mapper_config;
typedef struct { int n_corner, n_surf, map_corner, map_surf, cells_in_fov_corner, cells_in_fov_surf, appended_corner, appended_surf;
                 float ms_front_end, ms_refresh, ms_register, ms_append; /* host wall clock per phase, syncs included */ } ll_mapper_stats;
typedef struct ll_mapper ll_mapper;
void ll_mapper_config_default(ll_mapper_config* cfg);
int  ll_mapper_create(ll_ctx* ctx, const ll_mapper_config* cfg, ll_mapper** out);
void ll_mapper_release(ll_mapper* mapper);
/* One raw scan through process_new_scan (laser_mapping.hpp:1316-1521): features, match-map refresh from the cell maps, registration
 * (out->status 1 accepted/skipped, 0 rejected and discarded), world-frame features appended to the cell maps, pose adopted.
 * LL_ERR_INVALID for an unknown fmt or where or a null raw of n > 0 points, LL_ERR_CAPACITY for n over max_scan_points: nothing changed. */
int  ll_mapper_process_scan(ll_mapper* mapper, const void* raw, size_t n, int fmt, int where, double stamp, ll_reg_result* out, ll_mapper_stats* stats);
/* One sensor frame through Laser_feature::laserCloudHandler and, for every piece it publishes, Laser_mapping::process_new_scan
 * (laser_feature_extractor.hpp:305-389, laser_mapping.hpp:1316-1521): what the shipped configs run (common/odom_mode 1, if_motion_deblur 0).
 * n_heads (1 ... 8) raw clouds (Mid-100: 3), one extractor over the heads in turn as ll_frame_to_pose; a head with <= 5 petals contributes
 * nothing, and when no head contributes nothing is published (*n_pieces = 0, the mapper untouched).  The frame is cut into
 * pieces = reg.if_motion_deblur ? 1 : pipeline.pieces (1 ... 16) pieces of consecutive petals (pipeline.whole_frame and use_piece are not
 * read); piece i's features are the piece-i clouds of the contributing heads in head order, down-sampled by the extractor's and the mapping
 * node's VoxelGrids.  odom_mode 1 registers every piece as a scan of its own (frame index, time-stamp range, map refresh, append and pose
 * adoption per piece), 0 only piece 0.  out / stats (stats may be NULL) receive one entry per published piece; cap is their length.
 * LL_ERR_INVALID (nothing changed) for odom_mode outside {0, 1}, pieces outside 1 ... 16, cap below the pieces to publish, an unknown
 * fmt or where or a null cloud of points;
 * LL_ERR_CAPACITY up front when the heads exceed max_scan_points, and before piece i's registration when its features exceed max_features
 * (*n_pieces then counts the pieces completed, whose entries are valid). */
#define LL_MAX_PIECES_PER_FRAME 16
int  ll_mapper_process_frame(ll_mapper* mapper, int n_heads, const void* const* raws, const size_t* ns, int fmt, int where, const double* stamps,
                             int odom_mode, ll_reg_result* out, ll_mapper_stats* stats, int cap, int* n_pieces);
/* Sequences (recorded data replayed or mapped offline faster than real time): the front end of input k + 1 runs on the device, on streams of
 * the least priority (the context's own streams have the greatest), while input k is registered.  A live node gains nothing (the next frame does not exist yet) and keeps the single calls.
 *
 * ll_mapper_process_frames: n_frames frames of n_heads heads each, in order: the results of n_frames calls of ll_mapper_process_frame.
 * Frame f's heads are raws / ns / stamps [f * n_heads + h].  out / stats (stats may be NULL): cap entries per frame (out[f * cap + i] = piece i
 * of frame f); n_pieces[f] as the single call's *n_pieces.
 * ll_mapper_process_scans: n_scans raw scans, the results of n_scans calls of ll_mapper_process_scan (out[k], stats[k]).
 *
 * Identity: every entry equals the single call's in every ll_reg_result field except gpu_ms_*, and in every integer field of ll_mapper_stats;
 * ll_mapper_pose and the mapper and extractor state after the call equal the single calls' too.  ms_* stay host wall clock per phase;
 * ms_front_end is the time this call spent enqueuing and waiting for that input's front end, so it falls when the front end is hidden.
 * Validation first: null pointers, n_frames / n_scans < 1, n_heads outside 1 ... 8, an unknown fmt or where, a bad odom_mode, pieces or cap
 * (LL_ERR_INVALID) and any frame or scan over max_scan_points (LL_ERR_CAPACITY) are found for the whole sequence before anything is
 * enqueued; nothing changes then.  An error while running (a piece or scan over max_features: LL_ERR_CAPACITY; or an error of the single
 * call's registration) stops the sequence at input f: *n_frames_done / *n_scans_done = f, n_pieces[f] = the pieces of frame f completed, and
 * the mapper and the extractor's time bookkeeping are exactly as after the single calls up to and including the failing one, so the caller
 * can go on with input f + 1 by either API.  Inputs need only stay valid for the duration of the call; nothing is pending between calls. */
int  ll_mapper_process_frames(ll_mapper* mapper, int n_frames, int n_heads, const void* const* raws, const size_t* ns, int fmt, int where,
                              const double* stamps, int odom_mode, ll_reg_result* out, ll_mapper_stats* stats, int cap, int* n_pieces,
                              int* n_frames_done);
int  ll_mapper_process_scans(ll_mapper* mapper, int n_scans, const void* const* raws, const size_t* ns, int fmt, int where, const double* stamps,
                             ll_reg_result* out, ll_mapper_stats* stats, int* n_scans_done);
int  ll_mapper_pose(const ll_mapper* mapper, double q_wxyz[4], double t[3], int* frame_index);

/* ---- checkpoint: the whole streaming mapper as one byte image ------------------------------------------------------------------------
 * Stop a mapping run and resume it in another process or on another GPU, keep a map for the next session, move a stream between contexts.
 * A mapper restored from an image continues bit for bit as the one that was saved: every ll_reg_result field except gpu_ms_*, every integer
 * field of ll_mapper_stats and ll_mapper_pose.  (The reference persists its cell map as JSON, cell_map_keyframe.hpp:818-914; this is a
 * binary image of the whole mapper instead.)
 *
 * Format (version 1), one little-endian byte string:
 *   ll_mapper_image_header      magic "LLMAPIMG", version, config_bytes = sizeof(ll_mapper_config), total_bytes = the image's size, and
 *                               one (offset, length) per section, in the order of the LL_IMAGE_* indices below
 *   LL_IMAGE_CONFIG             the ll_mapper_config the mapper was created with, verbatim
 *   LL_IMAGE_SCALARS            ll_mapper_image_scalars
 *   LL_IMAGE_HISTORY_{CORNER,SURF}   the history window of one class (mode 0's match map):
 *                               int64 n_segments, int64 n_points, int32 size[n_segments] (oldest first), ll_point points[n_points] (window order)
 *   LL_IMAGE_SNAPSHOT_{CORNER,SURF}  the whole-map VoxelGrid output the current kNN index was built from (empty when have_map = 0):
 *                               int64 n, ll_point points[n]
 *   LL_IMAGE_CELLS_{CORNER,SURF}     one cell map: int32 current_frame_idx, int32 n_out_of_range, int64 n_cells, int64 n_points,
 *                               ll_image_cell cells[n_cells] (every cell of the table, also cells without a live point, in ascending key),
 *                               ll_image_cell_point points[n_points] (the live points only, in store order)
 * A writer places the sections back to back after the header in index order.  The image is canonical: it depends only on the mapper's
 * observable state, never on hash-slot placement, dead store entries, epochs, table capacity, reservations or arena offsets, so the same
 * stream gives byte-identical images and load-then-save reproduces an image byte for byte.  Front-end graphs and launch counters are not
 * saved (a restored mapper captures its graphs afresh).  Images are not portable across endianness. */
#define LL_MAPPER_IMAGE_MAGIC "LLMAPIMG"
#define LL_MAPPER_IMAGE_VERSION 1
enum { LL_IMAGE_CONFIG = 0, LL_IMAGE_SCALARS = 1, LL_IMAGE_HISTORY_CORNER = 2, LL_IMAGE_HISTORY_SURF = 3, LL_IMAGE_SNAPSHOT_CORNER = 4,
       LL_IMAGE_SNAPSHOT_SURF = 5, LL_IMAGE_CELLS_CORNER = 6, LL_IMAGE_CELLS_SURF = 7, LL_IMAGE_SECTIONS = 8 };
typedef struct { uint64_t offset, length; } ll_image_section;
typedef struct { char magic[8]; uint32_t version, config_bytes; uint64_t total_bytes; ll_image_section section[LL_IMAGE_SECTIONS]; } ll_mapper_image_header;   /* 152 B */
typedef struct {
  int32_t frame_index;                          /* m_current_frame_index                                                                  */
  int32_t map_dirty, have_map;                  /* 0 / 1: the match map is refreshed at the next step / the kNN index exists             */
  int32_t snap_n[2], fov[2];                    /* what the next ll_mapper_stats reports when map_dirty = 0 (map_*, cells_in_fov_*)      */
  int32_t reserved;                             /* 0                                                                                      */
  double  last_time_stamp;                      /* m_last_time_stamp                                                                      */
  double  q_w_curr[4], t_w_curr[3];             /* the pose                                                                               */
  double  last_his_add_q[4], last_his_add_t[3]; /* m_last_his_add_q / _t                                                                  */
  double  first_receive_time, current_time, last_maximum_time_stamp;   /* the context's extractor time bookkeeping                       */
} ll_mapper_image_scalars;                      /* 176 B */
typedef struct { uint64_t key; int32_t create_frame, last_update; } ll_image_cell;   /* key: cell index (k, j, i) + 2^20 in 21 bits each, k highest */
typedef struct { float x, y, z; int32_t cell; } ll_image_cell_point;               /* cell: index into the section's cell list */
typedef struct {
  uint64_t bytes;
  int64_t  history_points[2], snapshot_points[2], cells[2], cell_points[2];   /* [0] corner, [1] surface; cell_points: live points */
  uint32_t version;
  int32_t  matching_mode, frame_index, have_map, map_dirty;
  int32_t  history_segments[2], cell_frame_idx[2];
  int32_t  reserved;
} ll_image_info;                                /* 112 B */
/* image NULL: *bytes = the size needed.  cap < needed: LL_ERR_CAPACITY, nothing written (*bytes = the size needed).  The mapper is not modified. */
int  ll_mapper_save(ll_mapper* mapper, void* image, size_t cap, size_t* bytes);
/* A new mapper on ctx in the image's state.  cfg NULL: the image's config.  Otherwise cfg must equal it in every field except max_cells,
 * reserve_map_points and reserve_store_points (LL_ERR_INVALID), which size the new mapper's buffers only: its own images keep the image's
 * config, so that load-then-save reproduces the image byte for byte.  Sets ctx's extractor time bookkeeping,
 * as ll_mapper_create resets it.  The image is validated completely before anything touches the device: a refused image (LL_ERR_INVALID; a
 * cell map with more cells than half the table of the effective max_cells: LL_ERR_CAPACITY) creates nothing and changes nothing. */
int  ll_mapper_load(ll_ctx* ctx, const void* image, size_t bytes, const ll_mapper_config* cfg, ll_mapper** out);
/* Host only, no context or GPU: validates an image completely (as ll_mapper_load with cfg NULL) and reports what is in it. */
int  ll_mapper_image_info(const void* image, size_t bytes, ll_image_info* info);

/* ---- relocalization: a scan's pose in a prior map without an initial guess (beyond the reference; DESIGN.md §4.3) ------------------
 * Every other entry point needs a guess inside the basin of ICP (about the +-para_max_speed box and a few degrees).  These find one: an
 * occupancy index of the map, every hypothesis of a rotation set x translation lattice scored against it on the device, the first K local maxima
 * of the score (peaks) refined as the items of one ll_register_batch, the best accepted item chosen. */
typedef struct ll_reloc_index ll_reloc_index;
/* The occupancy index of `map` (not sharded: LL_ERR_INVALID), built from its own device clouds (corners and surfaces, finite points only).  The
 * anchor lo is the finite bounding box the map keeps; a point's cell on axis a is floor(((double)x_a - (double)lo_a) / (double)res) + dilate,
 * computed in fp64 and compared as a double before it becomes an integer; dims_a = floor(((double)hi_a - lo_a) / res) + 1 + 2 dilate.  A voxel is
 * set iff an occupied voxel lies within Chebyshev distance `dilate` of it.  res <= 0 (or not finite), dilate outside 0 ... 4 or max_hypotheses
 * outside 1 ... 2^24: LL_ERR_INVALID; more than 2^30 voxels: LL_ERR_CAPACITY; a map without a finite point: LL_ERR_INVALID; all before anything is
 * enqueued.  Everything a relocalization needs is allocated here once (the bitmask, 44 bytes per hypothesis of max_hypotheses, the score
 * points): ll_relocalize allocates nothing.  The index belongs to this map as it is now (ll_map_rebuild of it invalidates the index), and is used
 * by one call at a time. */
int  ll_reloc_index_build(ll_ctx* ctx, const ll_map* map, float res, int dilate, int max_hypotheses, ll_reloc_index** out);
void ll_reloc_index_release(ll_reloc_index* idx);
/* Parity hook: dims[3], lo[3] (the grid's fp32 anchor) and the dilated bitmask, voxel v = x + dims0 (y + dims1 z) in bit v & 31 of word v >> 5
 * (ceil(dims0 dims1 dims2 / 32) words; words NULL: only dims and lo; cap_words too small: LL_ERR_CAPACITY). */
int  ll_reloc_index_read(const ll_reloc_index* idx, int dims[3], float lo[3], uint32_t* words, size_t cap_words);
typedef struct {
  int           n_rot;  const double* rot_wxyz;   /* hypothesis rotations, host, n_rot x 4 (w,x,y,z), unit norm within 1e-6             */
  int           rot_cyclic;                       /* rotation r's neighbours are r-1 and r+1 mod n_rot (a yaw circle)                    */
  double        t0[3], step[3]; int nt[3];        /* translation lattice: t = t0 + i*step per axis, i in 0 .. nt-1                       */
  int           max_candidates;                   /* K, 1 .. LL_MAX_BATCH                                                                */
} ll_reloc_cfg;
typedef struct { double q_wxyz[4], t[3]; int32_t score, hypothesis; } ll_reloc_candidate;
/* Score points that ll_relocalize accepts at most (LL_ERR_CAPACITY above). */
#define LL_RELOC_MAX_SCORE_POINTS 8192
/* Hypothesis h = i + nt0 (j + nt1 (k + nt2 r)) (x fastest, rotation slowest) is the pose (rot_wxyz[r], t0 + (i, j, k) * step).  Its score is the
 * number of score points p (scan frame, finite xyz) whose p_w = (float)(q_r * p + t) (fp64 rotation, the association of ll_transform, rounded to
 * fp32 per component) falls on a set voxel inside the grid.  h is a peak iff score(h) >= 1 and h comes first in (score descending, index
 * ascending) among its lattice Chebyshev-1 neighbours (clipped at the border) at rotations r - 1, r, r + 1 (wrapped when rot_cyclic and
 * n_rot >= 3).  The candidates are the first K peaks in that order (*n_cand <= K of them, cand[0 .. *n_cand)).  Each is refined as one item of
 * ll_register_batch over corner / surf with tmpl, its q_w_last = q_w_curr and t_w_last = t_w_curr set to the candidate and
 * para_buffer_incremental to identity: refined[j] and item_status[j] are what ll_register_batch returns for it.  *best = the rank j with
 * item_status LL_OK, registered 1 and status 1 of the smallest inlier_threshold (:559, the score Scene_alignment uses), ties to the lower rank;
 * -1 when none qualifies (the call still returns LL_OK).  cand / refined / item_status hold max_candidates entries.
 * Before anything is enqueued: a null pointer, a non-unit quaternion, n_rot or nt < 1, more hypotheses than the index's max_hypotheses, K outside
 * 1 ... LL_MAX_BATCH, a sharded map, an index built on another map, an unknown fmt / where or a tmpl whose frame index is at or below
 * mapping_init_accumulate_frames (the :199 gate would skip every refinement): LL_ERR_INVALID; more than LL_RELOC_MAX_SCORE_POINTS score points,
 * or K items of these features failing the batch's capacity check: LL_ERR_CAPACITY. */
int ll_relocalize(ll_ctx* ctx, const ll_map* map, const ll_reloc_index* idx,
                  const void* score_pts, size_t n_score,
                  const void* corner, size_t n_corner, const void* surf, size_t n_surf, int fmt, int where,
                  const ll_reloc_cfg* cfg, const ll_reg_state* tmpl,
                  ll_reloc_candidate* cand, ll_reg_result* refined, int* item_status, int* n_cand, int* best);
/* Parity hook: the scores of all n_rot x nt0 x nt1 x nt2 hypotheses (hypothesis order), validated as ll_relocalize validates them. */
int ll_reloc_scores(ll_ctx* ctx, const ll_reloc_index* idx, const void* score_pts, size_t n_score, int fmt, int where,
                    const ll_reloc_cfg* cfg, int32_t* scores);

/* ---- relocalization by class-aware distance fields (DESIGN.md §4.3.1) -----------------------------------------------------------
 * The same search with a graded, class-aware score, a fine search around every candidate and a choice that sees the points an alias leaves
 * outside the map: coarse peaks of the field score, each refined by a fine lattice of its own, the fine picks registered as one
 * ll_register_batch, the accepted item of the largest field score at its refined pose chosen. */
typedef struct ll_reloc_field ll_reloc_field;
/* One truncated squared distance field per class of `map` (not sharded: LL_ERR_INVALID), from its own device clouds (finite points only).  The
 * grid is that of ll_reloc_index_build with T = trunc in place of dilate: lo the map's finite bounding-box minimum, a point's cell on axis a
 * floor(((double)x_a - (double)lo_a) / (double)res) + T in fp64, dims_a = floor(((double)hi_a - lo_a) / res) + 1 + 2 T.  D_c(v) = min(T^2, the
 * smallest squared voxel distance |u - v|^2 from v to a voxel u holding a point of class c), one byte per voxel (a class without a point: T^2
 * everywhere).  Built by three separable integer passes, so it is deterministic.  res <= 0 (or not finite), trunc outside 1 ... 15 or
 * max_hypotheses outside 1 ... 2^24: LL_ERR_INVALID; more than 2^30 voxels: LL_ERR_CAPACITY; a map without a finite point: LL_ERR_INVALID; all
 * before anything is enqueued.  Everything ll_relocalize_field needs is allocated here once (2 bytes per voxel, 48 bytes per hypothesis of
 * max_hypotheses, the score points of both classes): ll_relocalize_field allocates no device memory.  The field belongs to this map as it is now
 * (ll_map_rebuild of it invalidates the field), and is used by one call at a time. */
int  ll_reloc_field_build(ll_ctx* ctx, const ll_map* map, float res, int trunc, int max_hypotheses, ll_reloc_field** out);
void ll_reloc_field_release(ll_reloc_field* field);
/* Parity hook: dims[3], lo[3] and the field of class `which` (0 corner, 1 surface), voxel v = x + dims0 (y + dims1 z) in byte v (dims0 dims1 dims2
 * bytes; d2 NULL: only dims and lo; cap too small: LL_ERR_CAPACITY; which not 0 / 1: LL_ERR_INVALID). */
int  ll_reloc_field_read(const ll_reloc_field* field, int which, int dims[3], float lo[3], uint8_t* d2, size_t cap);
typedef struct {
  int           n_rot;  const double* rot_wxyz;   /* offsets dq, host, n_rot x 4 (w,x,y,z), unit norm within 1e-6                          */
  double        step[3]; int nt[3];               /* lattice per candidate: nt odd per axis, centred on the candidate's translation         */
} ll_reloc_fine_cfg;
typedef struct {
  double  q_wxyz[4], t[3]; int32_t score, hypothesis;                /* the coarse peak: pose, field score, hypothesis (as ll_reloc_candidate) */
  double  fine_q_wxyz[4], fine_t[3]; int32_t fine_score, fine_index; /* the fine pick: pose, field score, index r * n_lat + l in its group    */
  int32_t verify_score, reserved;                                    /* the field score at refined[j]'s pose; reserved = 0                   */
} ll_reloc_field_candidate;                                          /* 136 B */
/* The field score of pose (q, t): every score point p of class c with finite xyz, p_w = (float)(q * p + t) (fp64 rotation, the association of
 * ll_transform, rounded to fp32 per component) adds T^2 - D_c(cell(p_w)) when the cell is inside the grid, 0 otherwise; int32, corner points
 * read only the corner field and surface points only the surface field.
 * 1. Coarse: hypothesis h of `coarse` (as ll_relocalize) scored by the field score; the candidates are the first K = coarse->max_candidates peaks
 *    (the peak definition of ll_relocalize; *n_cand <= K of them).
 * 2. Fine: candidate j with pose (q_j, t_j) gets the group of rotations q_j (x) dq_r (Hamilton product in fp64, q_j on the left, each component
 *    summed left to right: w = w1 w2 - x1 x2 - y1 y2 - z1 z2, x = w1 x2 + x1 w2 + y1 z2 - z1 y2, y = w1 y2 - x1 z2 + y1 w2 + z1 x2,
 *    z = w1 z2 + x1 y2 - y1 x2 + z1 w2) times the lattice t = o_j + (i, j, k) * step, o_j = t_j - ((nt - 1) / 2) * step, fine index
 *    l + n_lat * r as in the coarse order.  Its pick is its first index in (score descending, index ascending).
 * 3. Refine: each pick seeds one item of ll_register_batch exactly as ll_relocalize seeds its candidates; refined[j] / item_status[j] are what
 *    the batch returns for it.
 * 4. Verify: cand[j].verify_score = the field score at (refined[j].q_w_curr, refined[j].t_w_curr).  *best = the rank j with item_status LL_OK,
 *    registered 1 and status 1 of the largest verify score, ties to the smaller inlier_threshold, then to the lower rank; -1 when none qualifies
 *    (the call still returns LL_OK).  cand / refined / item_status hold max_candidates entries.
 * Before anything is enqueued, everything ll_relocalize refuses (with this field in place of the index; more than LL_RELOC_MAX_SCORE_POINTS
 * score points in either class: LL_ERR_CAPACITY), and: a null fine cfg or fine rotation array, fine n_rot or nt < 1, an even fine nt, a
 * non-finite fine step, a non-unit dq, K x the fine hypotheses above max_hypotheses, a field on another device: LL_ERR_INVALID. */
int ll_relocalize_field(ll_ctx* ctx, const ll_map* map, const ll_reloc_field* field,
                        const void* score_corner, size_t n_score_corner, const void* score_surf, size_t n_score_surf,
                        const void* corner, size_t n_corner, const void* surf, size_t n_surf, int fmt, int where,
                        const ll_reloc_cfg* coarse, const ll_reloc_fine_cfg* fine, const ll_reg_state* tmpl,
                        ll_reloc_field_candidate* cand, ll_reg_result* refined, int* item_status, int* n_cand, int* best);
/* Parity hook: the field scores of all n_rot x nt0 x nt1 x nt2 hypotheses of cfg (hypothesis order), validated as ll_relocalize_field
 * validates them (max_candidates is not used). */
int ll_reloc_field_scores(ll_ctx* ctx, const ll_reloc_field* field, const void* score_corner, size_t n_score_corner, const void* score_surf,
                          size_t n_score_surf, int fmt, int where, const ll_reloc_cfg* cfg, int32_t* scores);
/* A new ll_map of the mapper's whole map: mode 0 = VoxelGrid (line / plane resolution) of the live history window, exactly what the next
 * refresh indexes; mode 1 = VoxelGrid of every live point of each cell map in store order (no FOV, no radius, no down-sample-and-replace).
 * The mapper's state does not change.  LL_ERR_INVALID when either class is empty (the mapper has no map yet).  Release with ll_map_release. */
int ll_mapper_whole_map(ll_mapper* mapper, ll_map** out);
/* The pose the next step seeds from (a relocalized pose, or any other).  Setting the pose the mapper already has (bitwise) changes nothing;
 * otherwise in matching mode 1 the match map is marked for refresh (the assembly is around the pose).  Frame index, time stamps and history
 * bookkeeping are untouched.  A non-finite value: LL_ERR_INVALID. */
int ll_mapper_set_pose(ll_mapper* mapper, const double q_wxyz[4], const double t[3]);

/* ---- tracking-loss recovery inside the streaming mapper (beyond the reference; DESIGN.md §4.3.2) -----------------------------------------
 * Off by default.  When on, every mapper step (every scan, every published piece of a frame, also inside the sequence calls) judges its own
 * registration: a registered step (registered 1) is bad when it is rejected (status 0) or its inlier_threshold (:559) exceeds
 * max_inlier_threshold.  A bad step is held back: nothing is appended and its pose is not adopted (as a rejected scan).  After lost_after
 * consecutive bad steps the mapper is lost; from then on every step registers as usual first, a good registration ends the loss, and a bad one
 * runs a relocalization of the step's own features in the mapper's own whole map (ll_relocalize_field's path):
 *   map     mode 0: the match map the mapper holds (the VoxelGrid of the live window, nothing appended since the first bad step); mode 1: the
 *           whole map of ll_mapper_whole_map rebuilt into a mapper-owned map.  The field is built once per loss episode.
 *   score   each class of the step's features through one VoxelGrid at score_leaf, the leaf doubled until a class fits
 *           LL_RELOC_MAX_SCORE_POINTS.
 *   coarse  the yaw circle of yaw_step_deg composed with the tilt of the mapper's pose (its yaw removed); the x / y lattice of t_step centred on
 *           the mapper's translation, half-width window_base + window_growth x the consecutive bad steps, clipped to the field's grid and to
 *           max_hypotheses; z the mapper's z.
 *   fine    yaw offsets +-yaw_step_deg / 2 at fine_yaw_step_deg, x / y +-fine_t_half coarse steps at fine_t_step (the Python defaults).
 *   adopt   best >= 0, verify_score / (T^2 (n_score_corner + n_score_surf)) >= min_verify_fraction and the refined inlier_threshold
 *           <= max_inlier_threshold: the pose is set as ll_mapper_set_pose sets it; the step itself is not appended.
 * The mapper's pose is the last good pose (or the last adopted one): the search is centred on it.  An attempt's error other than LL_ERR_CUDA is
 * logged and the step counts as bad; LL_ERR_CUDA is returned.  Recovery is a runtime setting: it is not part of a mapper image, and a loaded
 * mapper has it off until it is turned on again. */
typedef struct {
  double max_inlier_threshold;   /* the detection bound on inlier_threshold (m)                                                           */
  int    lost_after;             /* consecutive bad steps that make the mapper lost (>= 1)                                                */
  int    trunc;                  /* field truncation T (1 ... 15)                                                                         */
  float  res;                    /* field voxel (m)                                                                                       */
  float  score_leaf;             /* VoxelGrid leaf of the score points (m)                                                                */
  double yaw_step_deg, t_step;   /* coarse yaw step (deg, a divisor of 360 up to rounding) and translation step (m)                      */
  double window_base, window_growth;   /* lattice half-width (m) = window_base + window_growth x consecutive bad steps                    */
  int    max_candidates;         /* K, 1 ... LL_MAX_BATCH                                                                                 */
  int    max_hypotheses;         /* the field's hypothesis buffers (1 ... 2^24); must hold K x the fine hypotheses                        */
  double fine_yaw_step_deg, fine_t_step, fine_t_half;   /* fine search: yaw step (deg), translation step (m), half-width in coarse steps  */
  double min_verify_fraction;    /* adoption floor of verify_score / (T^2 x score points), 0 ... 1                                      */
  long long reserve_field_voxels;      /* field voxels allocated by ll_mapper_set_recovery                                                */
  long long reserve_whole_map_points;  /* mode 1: points per class of the whole map allocated by ll_mapper_set_recovery                   */
} ll_recovery_cfg;
void ll_mapper_recovery_default(ll_recovery_cfg* cfg);
/* cfg NULL: recovery off (its buffers released, the state back to tracking; the log keeps its entries).  Otherwise every value is checked
 * (LL_ERR_INVALID, the mapper unchanged) and everything an attempt needs is allocated now: the field (reserve_field_voxels, max_hypotheses),
 * the step's features and score points, the mode-1 whole map (reserve_whole_map_points).  Past these an attempt's buffers grow, and its log
 * entry says so.  Turning recovery on (again) starts in the tracking state. */
int  ll_mapper_set_recovery(ll_mapper* mapper, const ll_recovery_cfg* cfg);
enum { LL_TRACKING = 0, LL_SUSPECT = 1, LL_LOST = 2 };
enum { LL_BAD_NONE = 0, LL_BAD_REJECTED = 1, LL_BAD_INLIER = 2 };
/* One mapper step while recovery is on. */
typedef struct {
  int32_t frame_index;                 /* the registration's current_frame_index                                                        */
  int32_t state_before, state_after;   /* LL_TRACKING / LL_SUSPECT / LL_LOST                                                            */
  int32_t bad;                         /* LL_BAD_NONE, LL_BAD_REJECTED (status 0) or LL_BAD_INLIER (inlier_threshold over the bound)    */
  int32_t bad_steps;                   /* consecutive bad steps after this one                                                          */
  int32_t appended;                    /* 1 when the step's features were appended                                                     */
  int32_t attempted;                   /* 1 when a relocalization ran; the fields below describe it                                     */
  int32_t attempt_status;              /* LL_OK or the attempt's LL_ERR_*                                                               */
  int32_t nt[3], n_yaw;                /* the coarse lattice and yaw count                                                              */
  int32_t n_cand, best, adopted, grew; /* as ll_relocalize_field; adopted 1 when the pose was set; grew 1 when a buffer was reallocated */
  int32_t n_score[2];                  /* score points per class                                                                        */
  float   score_leaf[2];               /* the leaf each class was filtered with                                                         */
  double  t0[3], step[3];              /* the coarse lattice                                                                            */
  double  tilt_wxyz[4];                /* the tilt composed with the yaw circle                                                         */
  double  verify_fraction;             /* best's verify_score / (T^2 (n_score[0] + n_score[1])); 0 when best = -1                       */
  double  q_wxyz[4], t[3];             /* best's refined pose (the mapper's pose when best = -1)                                        */
  double  inlier_threshold;            /* best's refined inlier_threshold                                                               */
  double  ms_map, ms_search;           /* host wall clock: map + field build (0 when the episode's field was reused), the search        */
} ll_recovery_step;
#define LL_RECOVERY_LOG 1024
/* Drains up to cap entries, oldest first, from a ring of LL_RECOVERY_LOG entries (entries past cap stay for the next read).  *n_dropped = the
 * entries overwritten since the last read because the ring was full. */
int  ll_mapper_recovery_read(ll_mapper* mapper, ll_recovery_step* out, int cap, int* n, int* n_dropped);
/* Parity hook: what the last attempt passed to the search (LL_ERR_INVALID before any attempt).  n[4] = features (corner, surface) and score
 * points (corner, surface); coarse / fine as given to the search, rot_wxyz pointing at rot_coarse / rot_fine (n_rot x 4 each; NULL arrays:
 * counts only); tmpl = the step's registration state.  Point arrays hold cap_points, rotation arrays cap_rot rotations (LL_ERR_CAPACITY, nothing
 * written, when short). */
int  ll_mapper_recovery_last_inputs(ll_mapper* mapper, ll_reloc_cfg* coarse, ll_reloc_fine_cfg* fine, ll_reg_state* tmpl, size_t n[4],
                                    ll_point* corner, ll_point* surf, ll_point* score_corner, ll_point* score_surf, size_t cap_points,
                                    double* rot_coarse, double* rot_fine, int cap_rot);

/* ---- wire formats (SURVEY 8(f) N3)---------------------------------------------------------------------------------------------- */
/* Layout of one point record of an LL_FMT_STRIDED input: what pcl::fromROSMsg (laser_feature_extractor.hpp:275) resolves by field name from a
 * sensor_msgs/PointCloud2 (point_step, the offsets of the little-endian fields x, y, z, intensity and intensity's datatype).  The payload is
 * copied to the device as it is and unpacked there into 16-byte points; n = width * height. */
enum { LL_I_NONE = 0, LL_I_FLOAT32 = 7, LL_I_UINT8 = 2, LL_I_UINT16 = 4 };   /* = sensor_msgs/PointField datatype codes (0: no intensity field -> 0.0) */
typedef struct { int point_step, offset_x, offset_y, offset_z, offset_intensity, intensity_datatype; } ll_point_layout;
int  ll_set_point_layout(ll_ctx* ctx, const ll_point_layout* layout);
/* The output side (pcl::toROSMsg, laser_feature_extractor.hpp:367-384): the feature cloud of the last registration on this context (which = 0 corners,
 * 1 surfaces; what the feature node publishes on /pc2_corners, /pc2_surface) packed on the device into PointCloud2 records of the layout above.
 * out_host may be NULL to query *n_points first. */
int  ll_features_to_pointcloud2(ll_ctx* ctx, int which, void* out_host, size_t cap_bytes, size_t* n_points);
/* One accepted scan in the format of the reference's poses.log (laser_mapping.hpp:1506-1511; the Ceres BriefReport line is not reproduced).
 * Returns the number of characters written (excluding the terminating 0), or -1 when cap is too small. */
int  ll_format_pose_log(const ll_reg_result* r, char* buf, size_t cap);

/* Size of the registration-state snapshot copied to the host once per ICP iteration (for traffic accounting). */
int  ll_state_snapshot_bytes(void);
/* Diagnostics: cycle counters of the solver's master CTA over the last registration: eval, wait-for-slowest-CTA, grid reduce, lm_step, publish, #evaluations, staging, epilogue. */
int  ll_debug_solver_cycles(ll_ctx* ctx, long long out16[16]);   /* [8..12]: fused K10 section: L1 + insert, barrier, select, barrier, drop */

/* ---- device-to-device forms used when chaining stages without leaving the GPU (outputs in caller-provided device buffers) ------------- */
int ll_voxel_downsample_dev(ll_ctx* ctx, const ll_point* in_dev, size_t n, float leaf, ll_point* out_dev, size_t* n_out);
int ll_transform_dev(ll_ctx* ctx, const double q_wxyz[4], const double t[3], const ll_point* in_dev, size_t n, ll_point* out_dev);
/* Device pointers to the features of the last ll_register / ll_scan_to_pose on this context (scan frame, corners then surfaces). */
int ll_last_features_dev(ll_ctx* ctx, const ll_point** corner_dev, size_t* n_corner, const ll_point** surf_dev, size_t* n_surf);

/* ---- loop closure back end: the pose graph ----------------------------------------------------------- */
/* Replaces Ceres_pose_graph_3d::pose_graph_optimization (ceres_pose_graph_3d.hpp:282-352) as laser_mapping.hpp:1058-1089 calls it.
 * Poses 0 .. n-1; pose 0 is held constant (SetParameterBlockConstant on poses->begin()).  Edge (id_begin = a, id_end = b, t_be = (p^, q^),
 * information W): residual L [conj(q_a) (p_b - p_a) - p^ ; 2 vec(q^ (conj(q_a) q_b)^*)], L the lower Cholesky factor of W
 * (PoseGraph3dErrorTerm, :205-239).  Quaternions move by ceres' EigenQuaternionParameterization; the solver is ceres 1.14's
 * Levenberg-Marquardt trust region with Jacobi scaling, exact linear solves and max_num_iterations 200. */
typedef struct { double q_wxyz[4]; double t[3]; } ll_pose;
typedef struct { int id_begin, id_end; double q_wxyz[4]; double t[3]; double information[36]; /* row-major, symmetric positive definite */ } ll_pg_edge;
typedef struct {
  double initial_cost, final_cost;   /* 1/2 sum r^2 before, and the least cost an iteration reached (ceres' Summary) */
  int iterations, evaluations;       /* LM iterations (iteration zero not counted), residual + Jacobian evaluations */
  int termination;                   /* 0 iteration limit, 1 gradient, 2 parameter, 3 function tolerance, 4 failure (5 invalid steps), 5 radius */
  int border_nodes, segments, levels, free_nodes, reserved;   /* the elimination plan (see ll_pose_graph_optimize) */
  long long cycles_eval, cycles_elim, cycles_border, cycles_total;   /* SM clock cycles spent by the solve's phases (clock64) */
} ll_pg_summary;
/* Largest border the device solve accepts: the free endpoints of all loop edges (edges between non-consecutive free poses). */
#define LL_PG_MAX_BORDER 64
typedef struct ll_pose_graph ll_pose_graph;
/* A pose-graph solver on ctx's device and stream, with everything a solve of reserve_nodes poses and reserve_edges edges needs allocated now:
 * such a solve allocates no device memory; a larger one grows the buffers. */
int  ll_pose_graph_create(ll_ctx* ctx, int reserve_nodes, int reserve_edges, ll_pose_graph** out);
void ll_pose_graph_release(ll_pose_graph* pg);
/* Optimizes poses[0 .. n-1] in place (max_iterations <= 0: the reference's 200).  One kernel launch, the whole LM loop on the device:
 * odometry-chain segments are eliminated by block cyclic reduction, the border (free endpoints of the loop edges, at most LL_PG_MAX_BORDER,
 * else LL_ERR_CAPACITY) by a dense Cholesky factorization.  Poses no edge touches and pose 0 come back bit-unchanged.  m = 0 changes nothing
 * and reports 0 iterations.  LL_ERR_INVALID, with nothing changed or enqueued: an id outside 0 .. n-1, id_begin == id_end, a non-finite
 * value, an information matrix that is not symmetric positive definite. */
int  ll_pose_graph_optimize(ll_pose_graph* pg, ll_pose* poses, int n, const ll_pg_edge* edges, int m, int max_iterations, ll_pg_summary* summary);
/* Test hook: one LM step solve at the given poses and trust-region radius, with the Jacobi scaling s of these poses' Jacobian.  Per pose
 * (6 values: position, then rotation tangent; zero for poses that are not free): the gradient g = J^T r, the scaling s and the solution
 * `step` of (S J^T J S + D / radius) step = -S g, D = clamp(diag(S J^T J S), 1e-6, 1e32).  *valid = 0 when the factorization failed. */
int  ll_pose_graph_step(ll_pose_graph* pg, const ll_pose* poses, int n, const ll_pg_edge* edges, int m, double radius, double* cost, double* gradient,
                        double* scaling, double* step, int* valid);
/* The loop edge of Scene_alignment::add_constrain_of_loop (scene_alignment.hpp:97-127) with the inversion of laser_mapping.hpp:1065-1066:
 * icp = the pose ll_scene_align returned for the pair, a = the older keyframe (id_end), b = the newer one (id_begin).  icp is inverted
 * (Eigen's inverse(): conjugate / squared norm), then q = q_b^-1 icp^-1 q_a, t = q_b^-1 (icp^-1 (t_a - t_icp) - t_b), information = I. */
void ll_pose_graph_loop_edge(const double icp_q_wxyz[4], const double icp_t[3], const ll_pose* pose_a, int id_a, const ll_pose* pose_b, int id_b,
                             ll_pg_edge* out);
/* The corrected map the reference publishes after a loop closure (Mapping_refine::refine_pointcloud / refine_pts, ceres_pose_graph_3d.hpp:437-500,
 * its if_save == 0 path): keyframe k is clouds[seg_end[k - 1] .. seg_end[k]) (seg_end[-1] = 0), at most 256 keyframes per call.  Each keyframe is
 * down-sampled by a VoxelGrid at `leaf` (as ll_voxel_downsample_segments), then moved by the float transform R_aff p + T_aff with
 * R_aff = (R_opt R_ori^T) cast to float and T_aff = (double(R_aff) (-t_ori) + t_opt) cast to float (rotations by toRotationMatrix), from its pose
 * before (poses_ori[k]) and after (poses_opt[k]) the optimization.  The intensity of the output is 0.  out: the keyframes one after another
 * (at most n points), n_out_per_seg[k] their counts. */
int  ll_keyframes_repose(ll_ctx* ctx, const ll_point* clouds, size_t n, const size_t* seg_end, int n_kf, const ll_pose* poses_ori, const ll_pose* poses_opt,
                         float leaf, ll_point* out, size_t* n_out_per_seg);
/* R_aff (row-major) and T_aff of ll_keyframes_repose for one keyframe, as the host computes them. */
void ll_keyframe_affine(const ll_pose* pose_ori, const ll_pose* pose_opt, float R_aff[9], float T_aff[3]);

/* ---- loop detection: keyframes over the full-resolution cell map and the candidate search ------------------------------------------------ */
/* A keyframe (Maps_keyframe<float>, cell_map_keyframe.hpp:1002-1494) is a set of cells of one ll_cellmap, the caller's full-resolution map
 * (m_pt_cell_map_full, laser_mapping.hpp:617-618).  A cell here is one incarnation of a map cell: a revisit replaces a cell by an empty one
 * (find_cell, :716-758) and a keyframe that held the old one keeps it with its points.  Cells are ordered by ascending cell key (k, j, i), then
 * incarnation; that order replaces the reference's std::set of pointers (address order) in every sum and in the typed clouds.  A keyframe refers to
 * the map's point store: after a down-sample-and-replace assembly of the map, appends and analyses of the keyframes that held its cells before are
 * refused (LL_ERR_INVALID).  The accumulated cloud (m_accumulated_point_cloud) stays the caller's. */
typedef struct ll_keyframe ll_keyframe;
enum { LL_CELL_SPHERE = 0, LL_CELL_LINE = 1, LL_CELL_PLANE = 2, LL_CELL_ALL = -1 };   /* Feature_type (cell_map_keyframe.hpp:46-51); ALL: every cell */
typedef struct {
  int    cells, line_cells, plane_cells, accumulate_frames;
  float  center[3];                          /* get_center(): the mean of the cell centres (:1292-1302)                                     */
  float  roi_range;                          /* m_roi_range: 0.9 quantile of the distinct centre distances (:1304-1319); 0 without cells       */
  float  ratio_nonzero_line, ratio_nonzero_plane;   /* m_ratio_nonzero_*: image pixels >= 1 before the blur (:1423-1424)                    */
  size_t line_points, plane_points, all_points;     /* sizes of the typed clouds                                                          */
} ll_keyframe_info;
int  ll_keyframe_create(ll_ctx* ctx, ll_keyframe** out);
void ll_keyframe_release(ll_keyframe* kf);
/* laser_mapping.hpp:1527-1533: m_pt_cell_map_full.append_cloud(pts, &cell_vec), then add_cells(cell_vec) and m_accumulate_frames++ on each of the
 * n_open keyframes.  The append is ll_cellmap_append itself (same map state, same return codes); the cell set follows :585-665: every cell the
 * points reach on the first append into an empty map (set_point_cloud), afterwards the cells that received at least 3 of this call's points. */
int  ll_keyframe_append(ll_ctx* ctx, ll_cellmap* map, const void* pts, size_t n, int fmt, int where, ll_keyframe* const* open, int n_open);
/* Maps_keyframe::analyze (:1487-1494) over the keyframe's cells as `map` holds them now: per cell the mean and covariance (COMP_TYPE float,
 * IF_COV_INIT_IDENTITY 0, N - 1 divisor) and determine_feature (:436-473; sphere below 5 points or when |centre - mean| > 0.75 res, plane when
 * l1 / 3 > l0, line when l2 / 3 > l1, eigen-decomposition in fp64); then the centre, the ROI range, the 60 x 60 line / plane direction images
 * of generate_feature_img (:1385-1427) with their nonzero ratios, the Gaussian blur (9 x 9, sigma 4, wrap padding) and the typed clouds.
 * incremental_cov: common/if_update_mean_and_cov_incrementally of the map (1 in performance_precision.yaml, 0 in performance_realtime.yaml), one
 * value for the map's lifetime; the per-point recurrence of append_pt (:392-414) is replayed over each cell's points in append order. */
int  ll_keyframe_analyze(ll_ctx* ctx, ll_cellmap* map, ll_keyframe* kf, int incremental_cov, ll_keyframe_info* info);
int  ll_keyframe_get_info(const ll_keyframe* kf, ll_keyframe_info* info);
/* The analyzed keyframe's cells (at most cap): key (as ll_image_cell::key), incarnation, type and feature vector (3 floats; zero for spheres).
 * Any output may be NULL; *n = the keyframe's cell count.  keys and epochs are also available before an analysis. */
int  ll_keyframe_cells(ll_ctx* ctx, const ll_keyframe* kf, uint64_t* keys, int* epochs, int* types, float* vecs, int cap, int* n);
/* 60 x 60 row-major images [phi][theta]: direction counts before the blur and the blurred images; any may be NULL. */
int  ll_keyframe_images(ll_ctx* ctx, const ll_keyframe* kf, float* count_line, float* count_plane, float* line, float* plane);
/* extract_specify_points(e_feature_line / e_feature_plane) or get_all_pointcloud() (which = LL_CELL_LINE / LL_CELL_PLANE / LL_CELL_ALL,
 * :1263-1290): the points of those cells in cell order, append order inside a cell, intensity 0.  The cloud stays on the device (*out_dev, valid
 * until the next analysis of this keyframe), ready for ll_scene_align with LL_DEVICE; copied to out_host (cap points) when that is not NULL. */
int  ll_keyframe_cloud(ll_ctx* ctx, const ll_keyframe* kf, int which, ll_point* out_host, size_t cap, size_t* n_out, const ll_point** out_dev);
typedef struct {
  int   minimum_keyframe_differen;   /* loop_closure/minimum_keyframe_differen (200)                                                      */
  float avail_ratio_plane, avail_ratio_line;   /* laser_mapping.hpp:894-895 (0.05, 0.03)                                              */
  float maximum_roi_difference;      /* :1004 (5.0)                                                                                      */
  float minimum_similarity_linear, minimum_similarity_planar;   /* loop_closure/minimum_similarity_* (YAMLs: 0.65, 0.94)              */
  double plane_with_line;            /* :1012 (0.92, a double literal against the float similarity)                                      */
} ll_loop_cfg;
void ll_loop_cfg_default(ll_loop_cfg* cfg);
/* service_loop_detection's search (laser_mapping.hpp:988-1033) for kfs[newest] against kfs[0 .. newest - 1], every keyframe analyzed.  One launch
 * computes max_similiarity_of_two_image (matchTemplate CCORR_NORMED of the newest image against the earlier one wrap-padded by 30, max over
 * 61 x 61 positions) for the plane and the line images of every pair; sim_plane / sim_line[his] (newest entries, may be NULL).  candidates (his
 * ascending, at most newest) are the pairs that pass the keyframe-difference, nonzero-ratio, ROI-range (|d| > 5 in float), similarity and
 * cell-count gates; the cell-count gate is (a - b) / (a + b) * 0.1 in size_t (:1030), so a pair passes it only when the newest keyframe has at
 * least as many cells and the earlier one has some.  Alignment, `his += 10` (:1048-1052) and the stop after a true loop stay the caller's. */
int  ll_loop_search(ll_ctx* ctx, const ll_keyframe* const* kfs, int n, int newest, const ll_loop_cfg* cfg, float* sim_plane, float* sim_line, int* candidates,
                    int* n_candidates);

/* ---- loop closure inside the streaming mapper (loop_closure/if_enable_loop_closure; DESIGN.md §4.6) -------------------------------------
 * Off by default.  When on, every step whose features are appended (a rejected step, or one held back by recovery, does nothing here and does
 * not count as a frame) also runs Laser_mapping::process_new_scan's keyframe block (laser_mapping.hpp:1442, 1446-1459, 1480-1487, 1523-1564)
 * and, for a keyframe it closes, service_loop_detection (:874-1127), with every full cloud kept on the device:
 *   cloud   the step's full cloud (a scan: the front end's full cloud; a piece: the piece's full slices of every head, in head order), moved
 *           into the world by the registration pose (fp64, g_if_undistore = 0), pushed to the full history under the feature history's push
 *           condition and popped past maximum_history_size, appended to the mapper's full-resolution cell map (resolution and revisit
 *           threshold of the mapper's cell_resolution / threshold_cell_revisit, :617-618) and to every open keyframe (ll_keyframe_append).
 *   close   the front keyframe at scans_of_each_keyframe frames, with the mapper's pose after this step and its frame index (:1534-1543).
 *   open    when the back keyframe reaches scans_between_two_keyframe frames: the full history, VoxelGridded at surround_pointcloud_resolution,
 *           becomes that keyframe's accumulated cloud (:943-944 filters the same cloud later), the history is cleared and a keyframe opened.
 *   process a closed keyframe in the step that closes it: ll_keyframe_analyze, its pose and odometry edge, ll_loop_search over every earlier
 *           keyframe, the candidates in ascending order through ll_scene_align on the typed clouds (`his += 10` above twice the threshold, `his
 *           += 5` between the threshold and twice it, a loop below it), then ll_pose_graph_loop_edge, ll_pose_graph_optimize and the refined
 *           clouds of the published keyframes (pc_idx = n - 1, n - 3, ...; VoxelGrid 0.2, :903, and the affine of ll_keyframes_repose).
 * maximum_keyframe_in_waiting_list is not a setting: a closed keyframe is processed in the step that closes it, so the waiting list never holds
 * more than one and its pop (:1554-1557) cannot fire.  After the first loop the reference searches no more (if_end, :990-993): by default the
 * mapper then stops all loop-closure work; ll_mapper_set_loop_policy below lets it close further loops.  Loop closure never changes the
 * odometry: an error of its work other than LL_ERR_CUDA does not fail the step.
 * A failed alignment ends that keyframe's search (LL_LOOP_FAILED); any other error is logged (LL_LOOP_ERROR) and stops loop closure for good.
 * LL_ERR_CUDA is returned.  It is not part of a mapper image (a loaded mapper has it off): its state has an image of its own, the loop image
 * (ll_mapper_loop_save / ll_mapper_loop_load below). */
typedef struct {
  int    scans_of_each_keyframe;              /* loop_closure/scans_of_each_keyframe (300)                                                  */
  int    scans_between_two_keyframe;          /* loop_closure/scans_between_two_keyframe (100); must be < scans_of_each_keyframe           */
  ll_loop_cfg loop;                           /* the search's gates (minimum_keyframe_differen 200 in rosbag_loop.launch)                   */
  float  map_alignment_resolution;            /* loop_closure/map_alignment_resolution (0.1)                                                */
  int    map_alignment_maximum_icp_iteration; /* loop_closure/map_alignment_maximum_icp_iteration (5)                                      */
  float  map_alignment_inlier_threshold;      /* loop_closure/map_alignment_inlier_threshold (0.20)                                        */
  int    scene_alignment_maximum_residual_block;   /* loop_closure/scene_alignment_maximum_residual_block (3000)                           */
  double surround_pointcloud_resolution;      /* mapping/surround_pointcloud_resolution (0.30): the accumulated clouds' VoxelGrid leaf     */
  int    incremental_cov;                     /* common/if_update_mean_and_cov_incrementally (1)                                            */
  int    rng_seed;                            /* ll_align_cfg::rng_seed of every alignment                                                  */
  int    max_cells;                           /* the full map's cell table (as ll_cellmap_create; 0: its default; at most 2^29)            */
  long long reserve_map_points;               /* the full map's point store allocated by ll_mapper_set_loop_closure                        */
  long long reserve_history_points;           /* the full history allocated by ll_mapper_set_loop_closure                                  */
  int    reserve_keyframes;                   /* keyframes whose poses, edges and graph are allocated by ll_mapper_set_loop_closure        */
} ll_loop_closure_cfg;
/* The values rosbag_loop.launch runs: performance_precision.yaml with if_enable_loop_closure 1 and minimum_keyframe_differen 200. */
void ll_mapper_loop_closure_default(ll_loop_closure_cfg* cfg);
/* cfg NULL: loop closure off, its buffers and results released.  Otherwise every value is checked (LL_ERR_INVALID, the mapper unchanged;
 * scans_between_two_keyframe >= scans_of_each_keyframe is refused: the reference then calls back() on an empty keyframe list after a close),
 * everything the reservations cover is allocated, and loop closure starts again from an empty full map and one open keyframe (:626). */
int  ll_mapper_set_loop_closure(ll_mapper* mapper, const ll_loop_closure_cfg* cfg);
enum { LL_LOOP_KEYFRAME = 0, LL_LOOP_ALIGNMENT = 1, LL_LOOP_CLOSED = 2, LL_LOOP_ERROR = 3 };   /* ll_loop_event::kind                  */
enum { LL_LOOP_SKIP10 = 0, LL_LOOP_SKIP5 = 1, LL_LOOP_ACCEPT = 2, LL_LOOP_FAILED = 3 };   /* ll_loop_event::decision                          */
typedef struct {
  int32_t kind;                      /* LL_LOOP_KEYFRAME: a keyframe closed and processed; LL_LOOP_ALIGNMENT: one candidate aligned;
                                        LL_LOOP_CLOSED: the loop closed; LL_LOOP_ERROR: the loop work of the step ending at
                                        ending_frame_idx returned `status` (e.g. LL_ERR_CAPACITY of the full map's cell table) and loop
                                        closure stopped                                                                                  */
  int32_t keyframe;                  /* the newest keyframe's index (0, 1, ... in closing order)                                        */
  int32_t ending_frame_idx;          /* KEYFRAME: m_ending_frame_idx (the mapper's frame index after the closing step); ERROR: the step */
  int32_t n_candidates;              /* KEYFRAME: ll_loop_search's candidates (0 once the loop is closed)                               */
  ll_keyframe_info info;             /* KEYFRAME: ll_keyframe_analyze's result                                                          */
  double  q_wxyz[4], t[3];           /* KEYFRAME: the keyframe's pose                                                                   */
  int32_t his;                       /* ALIGNMENT, CLOSED: the earlier keyframe                                                         */
  int32_t scales_run;                /* ALIGNMENT: ll_scene_align's *scales_run                                                          */
  int32_t decision;                  /* ALIGNMENT: LL_LOOP_SKIP10, LL_LOOP_SKIP5, LL_LOOP_ACCEPT, or LL_LOOP_FAILED: ll_scene_align
                                        returned `status` (e.g. LL_ERR_CAPACITY: the typed clouds exceed max_features) and this keyframe's
                                        search ends there                                                                                */
  int32_t status;
  double  inlier_threshold;          /* ALIGNMENT: the alignment's inlier_threshold                                                     */
  double  icp_q_wxyz[4], icp_t[3];   /* ALIGNMENT: the alignment's pose                                                                 */
  ll_pg_edge edge;                   /* CLOSED: the loop edge                                                                           */
  ll_pg_summary summary;             /* CLOSED: ll_pose_graph_optimize's summary                                                        */
} ll_loop_event;
#define LL_LOOP_LOG 1024
/* Drains up to cap events, oldest first, from a ring of LL_LOOP_LOG (entries past cap stay); *n_dropped = events overwritten unread. */
int  ll_mapper_loop_read(ll_mapper* mapper, ll_loop_event* out, int cap, int* n, int* n_dropped);
/* The processed keyframes (*n, may be 0) and whether a loop is closed.  poses_ori: their poses (pose3d_map_ori); poses_opt: after the latest
 * optimization (temp_pose_3d_map) for the keyframes it covered (n_opt = the newest id of the latest loop edge + 1), the poses_ori values for
 * the others (all of them before a loop closes); edge: the latest loop edge (zeros before).  Arrays hold cap keyframes (LL_ERR_CAPACITY,
 * nothing written, when short); any may be NULL. */
int  ll_mapper_loop_result(ll_mapper* mapper, int* n, int* closed, ll_pose* poses_ori, ll_pose* poses_opt, int cap, ll_pg_edge* edge);
/* The refined cloud of published keyframe k of the latest optimization (after a loop closed; k = n_opt - 1, n_opt - 3, ..., else
 * LL_ERR_INVALID), as ll_keyframe_cloud offers its clouds: on the device (*out_dev, valid until the next loop closes or loop closure is set
 * again) and copied to out_host (cap points) when that is not NULL. */
int  ll_mapper_loop_cloud(ll_mapper* mapper, int k, ll_point* out_host, size_t cap, size_t* n_out, const ll_point** out_dev);
/* Loops after the first.  The reference stops after its first loop (if_end, :990-993), and so does the default policy {1, 0}.  With
 * max_loops = M > 1, loop closure goes on after a loop as before it (capture, history, full map, keyframes), with the same candidate walk, and
 * stops all work after the M-th loop.  A keyframe closed while newest - L < min_keyframes_between_loops (L: the newest keyframe of the last
 * loop) is analyzed and recorded but not searched (its LL_LOOP_KEYFRAME event has n_candidates 0).  Each loop adds its edge
 * (ll_pose_graph_loop_edge) to the loop edges so far; the graph of every odometry edge and every loop edge is solved from poses_ori, and every
 * keyframe up to the closing one is re-posed.  Accumulating loop edges goes beyond the reference, which solves one loop with only its edge.
 * M <= LL_MAX_LOOPS keeps every solve within LL_PG_MAX_BORDER; the graph of reserve_keyframes poses and reserve_keyframes - 1 + M edges is
 * allocated when the policy is set. */
#define LL_MAX_LOOPS (LL_PG_MAX_BORDER / 2)   /* 32: each loop edge adds at most two border poses */
typedef struct { int32_t max_loops, min_keyframes_between_loops; } ll_loop_policy;   /* 8 B */
void ll_mapper_loop_policy_default(ll_loop_policy* p);            /* {1, 0}: the reference (first loop, then stop) */
/* p NULL: the default.  LL_ERR_INVALID, nothing changed: loop closure off, a loop already closed, max_loops outside 1 ... LL_MAX_LOOPS, or
 * min_keyframes_between_loops < 0.  ll_mapper_set_loop_closure and ll_mapper_loop_load of a version-1 image reset the policy to the default. */
int  ll_mapper_set_loop_policy(ll_mapper* mapper, const ll_loop_policy* p);
/* Every loop edge so far, in closing order (*n_loops of them; edges may be NULL to query).  cap < *n_loops: LL_ERR_CAPACITY, nothing written. */
int  ll_mapper_loop_edges(ll_mapper* mapper, ll_pg_edge* edges, int cap, int* n_loops);

/* ---- loop feedback: the optimized trajectory back into the odometry (DESIGN.md §4.6.2) ----------------------------------------------------
 * Off by default, and then every output is what it is without this API.  With it on (matching mode 0), the step that closes a loop (its
 * LL_LOOP_CLOSED event) then moves the mapper onto the optimized trajectory:
 *   every live segment of both history windows (one step's world-frame features, frame index s) by A(s) o A_prev(s)^-1, where A is
 *           ll_loop_correction over this loop's poses and A_prev the same over the previous loop's (the identity before the first loop);
 *   the mapper's pose becomes the newest keyframe's optimized pose, the pose of the last window addition moves with the newest correction,
 *           and the next step rebuilds its match map from the moved window.
 * Loop closure stays in the odometry frame: with C the correction applied last (A of the latest loop at its newest keyframe, the identity
 * before a loop), it receives C^-1 o pose instead of the mapper's pose, for the step's full cloud and for the keyframe poses it records.  A
 * failure of the feedback other than LL_ERR_CUDA is checked before anything moves, logged as LL_LOOP_ERROR and stops loop closure.
 * Refused (LL_ERR_INVALID, nothing changed): loop closure off, a loop already closed, on = 1 in matching mode 1 (a cell-map point does not
 * record its step), maximum_history_size above LL_LOOP_FEEDBACK_MAX_SEGMENTS, or keyframes restored from a loop image of version 1 or 2
 * (their frame indices are not recorded there).  ll_mapper_set_loop_closure and ll_mapper_loop_load of such an image turn it off. */
#define LL_LOOP_FEEDBACK_MAX_SEGMENTS 4096   /* window segments the correction kernel stages in shared memory (both windows: 32 KiB) */
int  ll_mapper_set_loop_feedback(ll_mapper* mapper, int on);
/* C (q_wxyz, t) and how many corrections were applied.  Loop closure off: the identity and 0. */
int  ll_mapper_loop_correction_read(ll_mapper* mapper, double q_wxyz[4], double t[3], int* n_applied);
/* Host only, no context: the correction of the step with frame index s for keyframes 0 ... n - 1 closed at frame indices f[] (strictly
 * ascending), in fp64.  A_k = opt_k o ori_k^-1 (A_0 the identity: the graph holds pose 0 constant); A_0 for s <= f[0], A_(n-1) for
 * s >= f[n - 1], A_k at s = f[k], and between two keyframes, u = (s - f[k]) / (f[k + 1] - f[k]), the slerp of the rotations (the shorter arc)
 * and the linear interpolation of the translations.  LL_ERR_INVALID: a NULL array, n < 1 or f not strictly ascending. */
int  ll_loop_correction(const ll_pose* ori, const ll_pose* opt, const int* f, int n, int s, double q_wxyz[4], double t[3]);

/* ---- loop image: the mapper's loop closure as a byte image of its own (DESIGN.md §4.6.1) ------------------------------------------------
 * Checkpoint a run with loop closure on: save the mapper image and the loop image at the same step, then ll_mapper_load the one and
 * ll_mapper_loop_load the other onto the loaded mapper.  The restored mapper continues bit for bit as the saved one: every ll_reg_result field
 * except gpu_ms_*, every integer stat, every loop event (but ll_pg_summary::cycles_*, which time the solve and are saved as 0),
 * ll_mapper_loop_result and every ll_mapper_loop_cloud.  The mapper image is unchanged by loop closure (same bytes with it on or off).
 *
 * Format (version 1; version 2 differs in LL_LOOP_IMAGE_LOOP only), one little-endian byte string, with the mapper image's conventions (header of (offset, length) sections, placed back to
 * back in index order by a writer, canonical contents):
 *   ll_loop_image_header          magic "LLLOOPIM", version, config_bytes = sizeof(ll_loop_closure_cfg), total_bytes, the sections
 *   LL_LOOP_IMAGE_CONFIG          the ll_loop_closure_cfg in force, verbatim with its padding bytes zero
 *   LL_LOOP_IMAGE_SCALARS         ll_loop_image_scalars: the binding stamp, closed / stopped and the counts below
 *   LL_LOOP_IMAGE_CELLS           the full-resolution cell map: int32 current_frame_idx, int32 n_out_of_range, int64 n_cells, int64 n_points,
 *                                 ll_image_cell cells[n_cells] (ascending key), ll_image_cell_point points[n_points] (store order: the live
 *                                 points and those of every incarnation an open keyframe holds), int32 current[n_cells] (the ordinal of each
 *                                 cell's current incarnation), int32 incarnation[n_points] (each point's).  Ordinals number a cell's kept
 *                                 incarnations in epoch order: 0 is the cell's first incarnation (kept only while it exists), the later
 *                                 ones 1, 2, ...; so a cell has current + 1 kept incarnations when its first is kept, current otherwise
 *                                 (current <= current_frame_idx: a cell is replaced at most once per append).
 *   LL_LOOP_IMAGE_HISTORY         the full history: int64 n_segments, int64 n_points, int32 size[n_segments] (oldest first), ll_point points[]
 *   LL_LOOP_IMAGE_OPEN            the open keyframes in list order: ll_loop_image_open open[n_open], then each one's cells as
 *                                 ll_loop_image_ref (cell rank, incarnation ordinal), ascending
 *   LL_LOOP_IMAGE_KEYFRAMES       the closed keyframes in closing order: ll_keyframe_info info[n_keyframes]
 *   LL_LOOP_IMAGE_POSES           ll_pose poses_ori[n_keyframes]
 *   LL_LOOP_IMAGE_EDGES           ll_pg_edge odometry[n_keyframes - 1] (none without keyframes)
 *   LL_LOOP_IMAGE_IMAGES          float images[n_keyframes][4][60 * 60] (ll_keyframe_images' order; zeros for a keyframe without cells)
 *   LL_LOOP_IMAGE_CLOUDS          each closed keyframe's line then plane cloud (info.line_points + info.plane_points ll_point), in order
 *   LL_LOOP_IMAGE_ACCUMULATED     int64 n_acc (= n_keyframes + n_open - 1), int64 end[n_acc] (non-decreasing), ll_point points[end[n_acc - 1]]
 *   LL_LOOP_IMAGE_LOOP            closed = 1: ll_pg_edge loop_edge, ll_pose poses_opt[n_keyframes]; closed = 0: empty
 *                                 Version 2 (written under a policy other than the default, which writes version 1): always present,
 *                                 ll_loop_policy policy (max_loops >= 2), int32 n_loops (<= max_loops), int32 0, ll_pg_edge edges[n_loops]
 *                                 (closing order; their newest ids increase by at least min_keyframes_between_loops), ll_pose poses_opt[n_opt]
 *                                 (n_opt = the newest id of the last edge + 1, 0 without loops); closed = (n_loops > 0)
 *   LL_LOOP_IMAGE_EVENTS          the unread events, oldest first: ll_loop_event events[n_events] (n_events <= LL_LOOP_LOG), their
 *                                 summary.cycles_* (SM clock counters that time the solve, not state) 0
 * The refined clouds are not saved: ll_mapper_loop_load recomputes them from the accumulated clouds and both pose sets by the code the loop
 * ran.  Not saved either, as no result depends on them: the capture buffers (empty between calls), the pose-graph arena, hash slots, dead
 * incarnations no open keyframe holds, a closed keyframe's cell list, per-cell types and all-points cloud (only its info, images and line and
 * plane clouds are read again), capacities, reservations and arena offsets.  So the same stream gives byte-identical loop images, and
 * load-then-save reproduces one byte for byte.
 * The binding stamp (the mapper's frame index, pose, last time stamp, matching mode, and the mapper settings loop closure copied) guards
 * against pairing a loop image with the wrong mapper: ll_mapper_loop_load refuses an image whose stamp differs from the mapper's.  It is a
 * guard, not a proof that both images come from the same run and step. */
#define LL_LOOP_IMAGE_MAGIC "LLLOOPIM"
#define LL_LOOP_IMAGE_VERSION 1
#define LL_LOOP_IMAGE_VERSION_POLICY 2   /* the version a loop closure under a policy other than the default writes (LL_LOOP_IMAGE_LOOP above) */
/* Version 3, written with loop feedback on (whatever the policy): the header holds one more section, LL_LOOP_IMAGE_FEEDBACK, after the
 * thirteen; LL_LOOP_IMAGE_LOOP has version 2's layout with max_loops 1 ... LL_MAX_LOOPS.  LL_LOOP_IMAGE_FEEDBACK: int32 on (1), int32
 * n_applied (<= n_loops; < n_loops only when stopped), double c_q_wxyz[4], c_t[3] (the identity when n_applied is 0), int64 n_keyframes (the
 * scalars'), int64 n_segments, int32 f[n_keyframes] (each closed keyframe's frame index, strictly ascending), int32 frame[n_segments] (the
 * frame index of every live segment of the mapper's history windows, oldest first, strictly ascending).  Every frame index is within
 * 0 ... the stamp's frame_index, and ll_mapper_loop_load refuses the image unless n_segments equals the mapper's window segments. */
#define LL_LOOP_IMAGE_VERSION_FEEDBACK 3
enum { LL_LOOP_IMAGE_CONFIG = 0, LL_LOOP_IMAGE_SCALARS = 1, LL_LOOP_IMAGE_CELLS = 2, LL_LOOP_IMAGE_HISTORY = 3, LL_LOOP_IMAGE_OPEN = 4,
       LL_LOOP_IMAGE_KEYFRAMES = 5, LL_LOOP_IMAGE_POSES = 6, LL_LOOP_IMAGE_EDGES = 7, LL_LOOP_IMAGE_IMAGES = 8, LL_LOOP_IMAGE_CLOUDS = 9,
       LL_LOOP_IMAGE_ACCUMULATED = 10, LL_LOOP_IMAGE_LOOP = 11, LL_LOOP_IMAGE_EVENTS = 12, LL_LOOP_IMAGE_SECTIONS = 13,
       LL_LOOP_IMAGE_FEEDBACK = 13, LL_LOOP_IMAGE_SECTIONS_FEEDBACK = 14 };
typedef struct { char magic[8]; uint32_t version, config_bytes; uint64_t total_bytes; ll_image_section section[LL_LOOP_IMAGE_SECTIONS]; } ll_loop_image_header;   /* 232 B */
typedef struct {
  int32_t frame_index, matching_mode;           /* binding stamp: the mapper's m_current_frame_index and matching_mode,                  */
  int32_t threshold_cell_revisit, maximum_history_size, pieces;   /* its config values loop closure copied (pieces: pipeline.pieces)    */
  float   cell_resolution;
  double  last_time_stamp, q_w_curr[4], t_w_curr[3];   /* ... and its last time stamp and pose                                            */
  int32_t closed, stopped;                      /* 0 / 1: the loop closed (if_end) / an error stopped loop closure                        */
  int32_t n_keyframes, n_open, n_events, n_dropped;   /* closed keyframes, open keyframes (>= 1), unread events, events overwritten unread */
} ll_loop_image_scalars;                        /* 112 B */
typedef struct { int32_t frames, accumulate_frames; int64_t n_cells; } ll_loop_image_open;   /* frames since it opened, m_accumulate_frames */
typedef struct { int32_t cell, incarnation; } ll_loop_image_ref;                             /* cell rank in LL_LOOP_IMAGE_CELLS, ordinal   */
typedef struct {
  uint64_t bytes;
  int64_t  cells, cell_points;                  /* the full map's cells and kept points                                                   */
  int64_t  replaced_points;                     /* kept points of replaced incarnations (held by an open keyframe after a revisit)        */
  int64_t  history_points, cloud_points, accumulated_points;
  uint32_t version;
  int32_t  frame_index, matching_mode, closed, stopped, keyframes, open_keyframes, events, dropped;
  int32_t  max_incarnation;                     /* the largest current ordinal of a cell                                                  */
} ll_loop_image_summary;                         /* 96 B */
/* image NULL: *bytes = the size needed.  cap < needed: LL_ERR_CAPACITY, nothing written.  Loop closure off: LL_ERR_INVALID.  The mapper is not
 * modified (the event ring is not drained). */
int  ll_mapper_loop_save(ll_mapper* mapper, void* image, size_t cap, size_t* bytes);
/* Restores loop closure onto `mapper` (typically just made by ll_mapper_load from the mapper image saved at the same step), replacing any loop
 * closure it has, as ll_mapper_set_loop_closure does.  cfg NULL: the image's config; otherwise equal to it except max_cells and the reserve_*
 * fields, which size the allocations only (the mapper's later loop images keep the image's config).  The image is validated completely before
 * anything touches the device: a refused image (LL_ERR_INVALID; a stamp that differs from the mapper's: LL_ERR_INVALID; more cells than half
 * the table of the effective max_cells: LL_ERR_CAPACITY) changes nothing. */
int  ll_mapper_loop_load(ll_mapper* mapper, const void* image, size_t bytes, const ll_loop_closure_cfg* cfg);
/* Host only, no context or GPU: validates a loop image completely (as ll_mapper_loop_load with cfg NULL, but for the stamp and the cell table's
 * capacity: a mapper loaded with a larger max_cells can save an image that needs that max_cells again) and reports what is in it. */
int  ll_loop_image_info(const void* image, size_t bytes, ll_loop_image_summary* info);

/* ---- spinning-lidar front end: the Velodyne branch of Laser_feature::laserCloudHandler (DESIGN.md §4.7) ---------------------------------
 * laser_feature_extractor.hpp:393-825 with lidar_type other than "livox": NaN and near points removed (:399-400), ring and relative time per
 * point (:403-504), the rings concatenated (:510-521), curvature and neighbour flags (:524-598), per ring 6 sub-scans sorted by curvature with
 * the sharp and flat picks (:631-768), and the less-flat points VoxelGridded per ring at plane_resolution / 2 (:771-776).  Five clouds, in the
 * reference's push order: the full ring-ordered cloud (/laser_points_2, intensity = ring + 0.1 relTime), sharp (/laser_cloud_sharp), less
 * sharp, flat and less flat.  Stated deviations: the result is defined on the kept points (the reference reads past the filtered cloud when a
 * point was removed); the neighbour walks stop at the ends of the cloud; fewer than 5 kept points give empty feature clouds; a point with a
 * coordinate of magnitude above 1e36 is removed with the non-finite ones.  The 20-frame start-up delay (m_para_system_delay) is the caller's. */
typedef struct ll_spin ll_spin;
typedef struct {
  int   scan_line;          /* feature_extraction/scan_line: 16 or 64, anything else LL_ERR_INVALID (:160-164)                          */
  float minimum_range;      /* feature_extraction/minimum_range (0.1), the removeClosedPointCloud threshold                              */
  float plane_resolution;   /* feature_extraction/mapping_plane_resolution (0.4 in the shipped YAMLs): the less-flat VoxelGrid leaf is half */
  int   max_points;         /* input points per call the handle's arenas hold (the reference's per-point arrays: 400000)                 */
} ll_spin_cfg;
enum { LL_SPIN_FULL = 0, LL_SPIN_SHARP = 1, LL_SPIN_LESS_SHARP = 2, LL_SPIN_FLAT = 3, LL_SPIN_LESS_FLAT = 4 };
void ll_spin_cfg_default(ll_spin_cfg* cfg);
/* A spinning-lidar front end on ctx's device and stream, with its own arenas (ctx's footprint does not change); ctx must outlive it. */
int  ll_spin_create(ll_ctx* ctx, const ll_spin_cfg* cfg, ll_spin** out);
void ll_spin_release(ll_spin* spin);
/* One cloud through the front end: any input format (LL_FMT_STRIDED takes ctx's ll_set_point_layout), host or device.  counts[5] (may be
 * NULL): the sizes of the five clouds, indexed by LL_SPIN_*.  More than max_points: LL_ERR_CAPACITY, nothing changed.  One host
 * synchronisation, at the end. */
int  ll_spin_extract(ll_spin* spin, const void* raw, size_t n, int fmt, int where, size_t counts[5]);
/* Cloud `which` (LL_SPIN_*) of the last extract: on the device (*out_dev, valid until the next extract on this handle; the less-sharp and
 * less-flat clouds can go to ll_register / ll_map_build as LL_DEVICE inputs), copied to out_host (cap points) when that is not NULL. */
int  ll_spin_cloud(ll_spin* spin, int which, ll_point* out_host, size_t cap, size_t* n_out, const ll_point** out_dev);
/* Parity view of the full cloud's points (index order, cap entries; any array may be NULL): ring, curvature (0 outside [5, N - 5)), picked
 * before the selection (the occlusion and parallel-beam flags as they stand after :524-598) and the label (2 sharp, 1 less sharp, -1 flat, 0). */
int  ll_spin_point_info(ll_spin* spin, int32_t* ring, float* curvature, int32_t* picked, int32_t* label, size_t cap, size_t* n_out);
/* Diagnostics of the last extract: chains of the selection and the longest one in points. */
int  ll_spin_chains(const ll_spin* spin, int* n_chains, int* longest);

/* ---- streaming mapper on spinning-lidar sweeps (DESIGN.md §4.7.1) --------------------------------------------------------------------
 * The reference maps a Velodyne by remapping the feature node's /laser_cloud_less_sharp, /laser_cloud_less_flat and /laser_points_2 onto the
 * mapping node's /pc2_corners, /pc2_surface and /pc2_full.  ll_mapper_process_sweep is that pipeline in one call: the whole spin front end
 * (as ll_spin_extract), the mapping node's input VoxelGrids on the less-sharp cloud (pipeline.mapping_leaf_corner) and the less-flat cloud
 * (pipeline.mapping_leaf_surf), max_t = the largest intensity of the full cloud (-10000 when it is empty; there are no time stamps), then the
 * mapper step of ll_mapper_process_scan (refresh, registration, append, pose, recovery and loop closure).  Every sweep registers as one
 * scan: the frame index counts sweeps, and a sweep with fewer than 5 kept points goes through the step with 0 features (past the registration
 * gate that is LL_ERR_NO_BLOCKS, as for any empty scan: the frame index counted, nothing appended, the pose kept).  After a successful
 * call ll_spin_cloud gives the last sweep's five clouds, equal to ll_spin_extract's.  spin and mapper must share one context.
 * Refusals, with nothing changed: LL_ERR_INVALID for null pointers, n_sweeps < 1, an unknown fmt / where or a spin handle of another context;
 * LL_ERR_CAPACITY for a sweep over the handle's max_points or, with loop closure on, over the context's max_scan_points
 * (the full cloud loop closure takes from one step).
 * Features over max_features after the VoxelGrids: LL_ERR_CAPACITY before that sweep's registration (the mapper unchanged by it).
 * The 20-frame start-up delay (m_para_system_delay) stays the caller's. */
int  ll_mapper_process_sweep(ll_mapper* mapper, ll_spin* spin, const void* raw, size_t n, int fmt, int where, ll_reg_result* out, ll_mapper_stats* stats);
/* n_sweeps sweeps: the results of n_sweeps calls of ll_mapper_process_sweep (out[k], stats[k]; every field but gpu_ms_* and the float
 * timings), the front end of sweep k + 1 running under the step of sweep k.  Validated before anything is enqueued; an error at sweep f stops
 * there with *n_sweeps_done = f and the mapper as after the single calls up to f (ll_spin_cloud then has nothing extracted when sweep f + 1
 * had been enqueued ahead). */
int  ll_mapper_process_sweeps(ll_mapper* mapper, ll_spin* spin, int n_sweeps, const void* const* raws, const size_t* ns, int fmt, int where,
                              ll_reg_result* out, ll_mapper_stats* stats, int* n_sweeps_done);

/* ---- multi-GPU ------------------------------------------------------------------------------------- */
/* One process per GPU.  The 28-double normal equations (+4 counters) are all-reduced inside the solver kernel
 * through peer-mapped staging buffers (CUDA IPC over NVLink); the host only exchanges the IPC handles once. */
#define LL_IPC_HANDLE_BYTES 64
int ll_comm_local_handle(ll_ctx* ctx, unsigned char handle[LL_IPC_HANDLE_BYTES]);
int ll_comm_connect(ll_ctx* ctx, int rank, int world, const unsigned char* all_handles /* world x LL_IPC_HANDLE_BYTES */);

/* number of kernel launches issued by this context since creation (bench.py's gpu_launches) */
uint64_t ll_launch_count(const ll_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* LOAMLIVOX_B200_H */
