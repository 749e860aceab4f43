// Internal declarations shared by the CUDA translation units of libloamlivox_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <string>
#include <vector>
#include "../../include/loamlivox_b200.h"

#define LL_KNN 5

#define LL_CUDA(ctx, expr)                                                                        \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess) {                                                                      \
      (ctx)->set_error(std::string(#expr) + ": " + cudaGetErrorString(_e) + " @" + __FILE__ + ":" + std::to_string(__LINE__)); \
      return LL_ERR_CUDA;                                                                         \
    }                                                                                             \
  } while (0)
#define LL_TRY(expr) do { int _s = (expr); if (_s != LL_OK) return _s; } while (0)

// The layout of one device arena, written once: a layout function calls take() once per sub-array, in order.  Run on Carve() (null base) it
// only counts the bytes; run on Carve(base) it also assigns the pointers.  Sub-arrays start on 256-byte boundaries.
struct Carve {
  char* base = nullptr; size_t bytes = 0;
  Carve() = default;
  explicit Carve(void* b) : base((char*)b) {}
  template <typename T> T* take(size_t count) {
    char* r = base ? base + bytes : nullptr;
    bytes += (count * sizeof(T) + 255) & ~(size_t)255;
    return (T*)r;
  }
};
// Bytes of the layout `f` (a callable taking Carve&).
template <typename F> size_t layout_bytes(F&& f) { Carve c; f(c); return c.bytes; }

// Order-preserving float <-> int encoding: for non-NaN floats, int order == float order, so box bounds reduce with integer atomicMin / atomicMax.
__host__ __device__ inline int ll_f2ord(float f) {
#ifdef __CUDA_ARCH__
  const int i = __float_as_int(f);
#else
  int i; memcpy(&i, &f, 4);
#endif
  return i >= 0 ? i : i ^ 0x7fffffff;
}
__host__ __device__ inline float ll_ord2f(int i) {
  i = i >= 0 ? i : i ^ 0x7fffffff;
#ifdef __CUDA_ARCH__
  return __int_as_float(i);
#else
  float f; memcpy(&f, &i, 4); return f;
#endif
}

// ------------------------------------------------------------------------------------------------ device arrays
struct DevBuf {  // grow-only device allocation
  void* p = nullptr; size_t cap = 0;
  size_t floor = 0;   // smallest size ever allocated: a caller that knows how far the buffer will grow (the streaming mapper) sets it once, then nothing is
                      // reallocated in steady state (a cudaMalloc + cudaFree pair in a process with live streams and graphs stalls the call that triggers it)
  cudaError_t reserve(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    // first allocation: a little slack; regrowth: at least double, so that a buffer following a growing map is reallocated O(log n) times
    // (cudaFree synchronises the device)
    size_t want = bytes + bytes / 8 + 256;
    if (want < ((size_t)8 << 20)) want = (size_t)8 << 20;   // floor: every (re)allocation stalls the device, 8 MB of an 80 GB HBM costs nothing
    if (p && want < 2 * cap) want = 2 * cap;
    if (want < floor) want = floor;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    cudaError_t e = cudaMalloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
  cudaError_t reserve_floor(size_t bytes) { if (bytes > floor) floor = bytes; return reserve(floor); }   // allocate the floor now
  template <typename T> T* as() const { return (T*)p; }
  // Grows the buffer to the layout `f` (a callable taking Carve&), then assigns the layout's pointers inside it.
  template <typename F> cudaError_t carve(F&& f) {
    const cudaError_t e = reserve(layout_bytes(f));
    if (e == cudaSuccess) { Carve c(p); f(c); }
    return e;
  }
};

// ------------------------------------------------------------------------------------------------ map index
// "Bucket tree": map points sorted along a Hilbert curve (isotropic cells, 3 x 5..21 key bits: the width follows the map size), cut into
// leaf buckets of 32 points (512 B = one coalesced warp load), with a 32-ary tree of axis-aligned boxes above them (a node record = its 32
// children's boxes, 1 KB).  Search is exact: a box gives a true lower bound of the fp32 distance.  lo[l] holds level l's node records
// (the node array is laid out top level first).
#define LL_MAX_LEVELS 8
struct BucketTree {
  int n = 0;             // points given (the count of finite ones stays on the device)
  int n_pad = 0;         // padded to a multiple of 32
  int n_levels = 0;      // number of box levels (>= 1 when n > 0)
  int level_count[LL_MAX_LEVELS] = {0};   // boxes per level (unpadded)
  float4* pts = nullptr;                  // [n_pad] x,y,z, w = __int_as_float(original index); pad = +inf
  float4* lo[LL_MAX_LEVELS] = {nullptr};  // [level_count x 64] node records: child c of node j = rec[2c] (min xyz), rec[2c + 1] (max xyz), rec = lo[l] + 64 j
  float4* src = nullptr;                  // [n_src] the cloud as given to ll_map_build (x,y,z,intensity)
  int n_src = 0;
  float* d_bbox = nullptr;                // device: min xyz, max xyz of the finite points (6 floats inside `storage`)
  DevBuf storage;                          // one allocation backing all of the above
};

// Regular grid of cubic cells over the bounding box of the whole map (shard.cu): cell of a point = clamp(floor((p - origin) * inv_cell), 0, dims - 1)
// per axis, i.e. the border cells extend outwards without bound and every point of space has exactly one cell.
struct ShardGrid { float origin[3] = {0, 0, 0}; float cell = 1.f, inv_cell = 1.f; int dims[3] = {1, 1, 1}; };
__host__ __device__ inline int shard_cell_index(const ShardGrid& g, float x, float y, float z) {
  const float c[3] = {x, y, z}; int ci[3];
  for (int k = 0; k < 3; k++) { int v = (int)floorf((c[k] - g.origin[k]) * g.inv_cell); ci[k] = v < 0 ? 0 : (v > g.dims[k] - 1 ? g.dims[k] - 1 : v); }
  return (ci[2] * g.dims[1] + ci[1]) * g.dims[0] + ci[0];
}

struct ll_map {
  int device = 0;
  BucketTree corner, surf;
  // sharding (world == 1: everything owned).  A sharded snapshot indexes only the points of the cells this rank owns plus the halo of the match
  // gates around them; the owner table (rank per cell) lives on the device for the query side and on the host for ll_map_shard_info.
  int rank = 0, world = 1; float cell_size = 0.f;
  ShardGrid grid; float halo[2] = {0.f, 0.f}; DevBuf shard_owner; std::vector<int> h_owner; long long shard_total[2] = {0, 0};
};

// per-scan feature-extraction state (device)
struct ExtractState {
  int n = 0;
  float4* raw = nullptr;          // [n] x,y,z,reflectivity
  int* pt_type = nullptr; int* pt_label = nullptr;
  float* curvature = nullptr; float* view_angle = nullptr; float* depth_sq2 = nullptr; float* time_stamp = nullptr;
  float* polar_dis_sq2 = nullptr; int8_t* polar_dir = nullptr; uint8_t* self_mask = nullptr; uint8_t* cand = nullptr;
  int* cand_idx = nullptr; int* d_num_cand = nullptr;
  int* split_idx = nullptr;        // [<= n]
  int* scan_first = nullptr; int* scan_last = nullptr;
  double* d_time = nullptr;        // m_current_time of this scan (device scalar read by ex_point_kernel)
  int* d_meta = nullptr;           // [0]=n_split [1]=n_scans [2]=clutter_size
  double first_receive_time = -1, current_time = 0, last_maximum_time_stamp = 0;
};

// Registration arrays (device, one arena sized for max_features / max_scan_points at context creation)
struct RegArrays {
  float4* feat; float4* blk_a; double* blk_v; double* l1; double* k10_value;
  int* k10_n_distinct; int* knn_idx; float* knn_d; int* perm; float4* tmp_a; float4* tmp_b; float4* tmp_c; float4* tmp_d; int* counts; float* bounds;
};

// Solver / registration device state shared between kernels (lives in global memory)
struct RegDevState;  // defined in kernels.cuh
struct PinnedStage;  // pinned host staging of the small transfers (kernels.cuh)

// Timing events of a registration (ll_reg_result::gpu_ms_*): [0] start, [1] end
#define LL_TIMED_ITERS 16
struct RegEvents {
  cudaEvent_t total[2] = {nullptr, nullptr}, knn_first[2] = {nullptr, nullptr}, sort[2] = {nullptr, nullptr};
  cudaEvent_t phase[LL_TIMED_ITERS][5] = {};   // per ICP iteration, the bounds of its phases: kNN, solve #1, inlier select, solve #2
  template <typename F> void each(F&& f) {
    for (cudaEvent_t* g : {total, knn_first, sort}) { f(g[0]); f(g[1]); }
    for (auto& it : phase) for (cudaEvent_t& e : it) f(e);
  }
};
// Ordering events of the side streams (no timing)
struct SyncEvents {
  cudaEvent_t fork = nullptr, join = nullptr;     // stream <-> stream2
  cudaEvent_t fork3 = nullptr, join3 = nullptr;   // stream <-> stream3
  cudaEvent_t it[2] = {nullptr, nullptr};         // ICP iteration `it` has been snapshot into PinnedStage::snap[it & 1]
  template <typename F> void each(F&& f) { for (cudaEvent_t* e : {&fork, &join, &fork3, &join3, &it[0], &it[1]}) f(*e); }
};

struct ll_ctx {
  int device = 0;
  ll_config cfg;
  cudaStream_t stream = nullptr;
  RegEvents ev;
  SyncEvents sev;
  std::string err;
  uint64_t launches = 0;
  int hook_slots = 0;      // slot count left behind by ll_build_blocks / ll_set_blocks for the parity hooks
  int hook_cap_check = 0;  // ll_set_blocks: the slots exceed the state's residual-block cap (ll_solve_fused applies the drop rule, as a registration does)
  int last_nc = 0, last_ns = 0;   // features of the last registration (ll_last_features_dev)
  float last_full_min_t = 10000.f, last_full_max_t = -10000.f;   // find_min_max_intensity over the last front end's full cloud (laser_mapping.hpp:1336)
  int num_sms = 0;
  // arenas.  Sized at creation from the config, never moved afterwards: extract_buf, reg_buf and the front end's fe_*.
  DevBuf scratch;      // stream: CUB temporaries, the K10 hash set, the query sort, the index build and VoxelGrids of the map side
  DevBuf scratch2;     // stream2: the same for the corner half of the map side (index build, whole-map / append VoxelGrids, shard build)
  DevBuf fe_main, fe_corner, fe_petals;   // the front end's arenas on stream / stream2 / stream3 (what its captured graph touches)
  DevBuf stage_in;     // raw uploads (PCL32 or XYZI16)
  ll_point_layout layout = {16, 0, 4, 8, 12, LL_I_FLOAT32};   // LL_FMT_STRIDED records
  DevBuf extract_buf;  // ExtractState arrays
  DevBuf feat_buf;     // uploads and results of the cloud entry points (ll_voxel_downsample, ll_transform, ll_knn, host-side map builds)
  DevBuf reg_buf;      // RegArrays
  RegArrays A;
  PinnedStage* pin = nullptr;   // pinned host staging of the small H2D / D2H transfers
  ExtractState ex;
  RegDevState* d_reg = nullptr;   // device
  struct SolveSync* d_sync = nullptr;   // device: exchange rows of the solver kernels (solve.cu)
  // multi-GPU
  int rank = 0, world = 1;
  cudaStream_t stream2 = nullptr;   // side stream: the corner halves of the front end and of the map side
  cudaStream_t stream3 = nullptr;   // second side stream: the petal bookkeeping of the extractor (whole_frame front end)
  // The per-scan front end (extract + get_features + 4 VoxelGrids + count read-back) replayed as ONE CUDA graph: ~60 launches whose
  // enqueue cost on the host (CUB dispatch included) was longer than their execution.  Every buffer it touches is fixed at creation, so it is
  // re-captured only when the scan size or the pipeline config changes.
  struct FrontGraph { cudaGraphExec_t exec = nullptr; size_t n = 0; ll_pipeline_cfg pc; bool warm = false; uint64_t launches = 0; } fg;
  int reg_deblur = 0;                      // if_motion_deblur of the registration whose blocks are on the device
  int solve_world = 1;                     // world size the solver kernels all-reduce over (1 unless the map in use is sharded)
  void* comm_local = nullptr;              // this rank's staging slot (device memory, IPC-exported)
  void* comm_peers[8] = {nullptr};         // mapped peer slots (index = rank)
  void set_error(const std::string& s) { err = s; }
};

inline int ll_div_up(int a, int b) { return (a + b - 1) / b; }

// Residual-block cap (point_cloud_registration.hpp:232-238,339-345,434-458): the reference draws from a std::random_device-seeded mt19937
// (include/tools/tools_random.hpp:18-25).  The rule is kept, the numbers come from a counter-based generator keyed on the caller's seed
// (ll_reg_state::rng_seed), the ICP iteration, a stream (0 corner pre-skip, 1 surface pre-skip, 2 drop) and the feature / slot index:
// splitmix64 finaliser, top 24 bits -> float in [0,1).  Exported as ll_cap_uniform so that a test can pin it.
__host__ __device__ inline float ll_cap_uniform_f(int seed, int icp_iter, int stream, int index) {
  unsigned long long z = (unsigned long long)(unsigned)seed * 0x9E3779B97F4A7C15ull + (((unsigned long long)(unsigned)icp_iter << 40) | ((unsigned long long)(unsigned)stream << 32) | (unsigned long long)(unsigned)index);
  z ^= z >> 30; z *= 0xbf58476d1ce4e5b9ull; z ^= z >> 27; z *= 0x94d049bb133111ebull; z ^= z >> 31;
  return (float)(z >> 40) * (1.0f / 16777216.0f);
}
