// Map index ("bucket tree") build and the exact 5-NN search + residual-block construction kernels.
//
// Replaces, on the reference side:
//   pcl::KdTreeFLANN::setInputCloud            loam_livox/source/laser_mapping.hpp:544-545,
//                                              loam_livox/source/point_cloud_registration.hpp:596-597   (K5)
//   pointAssociateToMap + nearestKSearch(k=5)  loam_livox/source/point_cloud_registration.hpp:247-249,349-351,622-661 (K6)
//   gates + functor constructors               loam_livox/source/point_cloud_registration.hpp:254-331,353-431,
//                                              loam_livox/source/ceres_icp.hpp:246-260,314-336          (K7)
//
// Compiled with -fmad=false: the float distance (FLANN L2_Simple<float>: ((dx*dx)+dy*dy)+dz*dz), the fp64
// transform and the fp64 line/plane geometry must round exactly like the scalar CPU code.
#include <cub/cub.cuh>
#include <cstring>
#include <cstdlib>
#include "common.cuh"
#include "kernels.cuh"
#include "exact_math.cuh"

#define FULL 0xffffffffu
#define BUCKET 32     // points per leaf bucket: one per lane of the query's warp
#define FANOUT 32     // children per node; a node record holds its 32 children's boxes, child c = rec[2c] (lo.xyz) + rec[2c+1] (hi.xyz): 1 KB
#define NODE_F4 64    // float4s per node record
static_assert(BUCKET == 32 && FANOUT == 32 && NODE_F4 == 2 * FANOUT, "the search maps one bucket point / one child box to each lane of a warp");

// ------------------------------------------------------------------------------------------------ build
// bbox[0..2] = min (ll_f2ord encoding), bbox[3..5] = max, bbox[6] = number of finite points
__global__ void bbox_kernel(const float4* __restrict__ src, int n, int* __restrict__ bbox) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  int cnt = 0;
  for (; i < n; i += gridDim.x * blockDim.x) {
    float4 p = src[i];
    if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
      lo[0] = fminf(lo[0], p.x); lo[1] = fminf(lo[1], p.y); lo[2] = fminf(lo[2], p.z);
      hi[0] = fmaxf(hi[0], p.x); hi[1] = fmaxf(hi[1], p.y); hi[2] = fmaxf(hi[2], p.z);
      cnt++;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int k = 0; k < 3; k++) { lo[k] = fminf(lo[k], __shfl_xor_sync(FULL, lo[k], o)); hi[k] = fmaxf(hi[k], __shfl_xor_sync(FULL, hi[k], o)); }
    cnt += __shfl_xor_sync(FULL, cnt, o);
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < 3; k++) { atomicMin(&bbox[k], ll_f2ord(lo[k])); atomicMax(&bbox[3 + k], ll_f2ord(hi[k])); }
    atomicAdd(&bbox[6], cnt);
  }
}
__global__ void bbox_init_kernel(int* bbox) {
  if (threadIdx.x < 3) bbox[threadIdx.x] = ll_f2ord(INFINITY);
  else if (threadIdx.x < 6) bbox[threadIdx.x] = ll_f2ord(-INFINITY);
  else if (threadIdx.x == 6) bbox[6] = 0;
}

__device__ __forceinline__ unsigned long long spread21(unsigned v) {
  unsigned long long x = v & 0x1fffffull;
  x = (x | x << 32) & 0x1f00000000ffffull;
  x = (x | x << 16) & 0x1f0000ff0000ffull;
  x = (x | x << 8) & 0x100f00f00f00f00full;
  x = (x | x << 4) & 0x10c30c30c30c30c3ull;
  x = (x | x << 2) & 0x1249249249249249ull;
  return x;
}
// Hilbert index (Skilling's transpose form, `bits` per axis, <= 21) of the finite point c on an ISOTROPIC grid over the box lo..hi (one scale
// for all axes, the box's longest side), axes interleaved x first: < 2^(3 bits).  Consecutive runs along a Hilbert curve are connected blobs.
__device__ __forceinline__ unsigned long long hilbert_key(const float c[3], const float lo[3], const float hi[3], int bits) {
  const float ext = fmaxf(fmaxf(hi[0] - lo[0], hi[1] - lo[1]), hi[2] - lo[2]);
  const float scale = (float)(1u << bits), top = scale - 1.0f;
  unsigned X[3];
#pragma unroll
  for (int k = 0; k < 3; k++) {
    float u = ext > 0.f ? (c[k] - lo[k]) / ext : 0.f;
    u = fminf(fmaxf(u, 0.f), 1.f);
    X[k] = (unsigned)fminf(u * scale, top);
  }
  for (unsigned Q = 1u << (bits - 1); Q > 1; Q >>= 1) {
    const unsigned P = Q - 1;
#pragma unroll
    for (int k = 0; k < 3; k++) {
      if (X[k] & Q) X[0] ^= P;
      else { unsigned t = (X[0] ^ X[k]) & P; X[0] ^= t; X[k] ^= t; }
    }
  }
  X[1] ^= X[0]; X[2] ^= X[1];
  unsigned t = 0;
  for (unsigned Q = 1u << (bits - 1); Q > 1; Q >>= 1) if (X[2] & Q) t ^= Q - 1;
  X[0] ^= t; X[1] ^= t; X[2] ^= t;
  return (spread21(X[0]) << 2) | (spread21(X[1]) << 1) | spread21(X[2]);
}
// Map keys: fixed-size buckets of consecutive points get tight, nearly cubic boxes.  The key only decides WHICH points share a bucket (the
// boxes are computed from the points themselves, so the search is exact for any key): its width follows the map size (about 8 cells per bucket
// side at the finest level), which is what bounds the number of radix passes of the sort below.
template <typename KeyT>
__global__ void hilbert_kernel(const float4* __restrict__ src, int n, const int* __restrict__ bbox, int bits, KeyT* __restrict__ keys, int* __restrict__ vals) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float4 p = src[i];
  unsigned long long key = 1ull << (3 * bits);   // non-finite points: one bit above every real key -> they sort to the end
  if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
    const float lo[3] = {ll_ord2f(bbox[0]), ll_ord2f(bbox[1]), ll_ord2f(bbox[2])}, hi[3] = {ll_ord2f(bbox[3]), ll_ord2f(bbox[4]), ll_ord2f(bbox[5])};
    const float c[3] = {p.x, p.y, p.z};
    key = hilbert_key(c, lo, hi, bits);
  }
  keys[i] = (KeyT)key;
  vals[i] = i;
}
// n_valid (= bbox[6], the number of finite points) is read on the device: the host never waits for it.
__global__ void gather_kernel(const float4* __restrict__ src, const int* __restrict__ order, const int* __restrict__ bbox, int n_pad, float4* __restrict__ pts) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pad) return;
  const int n_valid = bbox[6];
  if (i < n_valid) { int j = order[i]; float4 p = src[j]; p.w = __int_as_float(j); pts[i] = p; }
  else pts[i] = make_float4(INFINITY, INFINITY, INFINITY, __int_as_float(0x7fffffff));
}
// One thread per (node, child).  Level 0: the children are buckets of 32 points (pad points are +inf and do not count).  Level l > 0: the children
// are level l-1 nodes (box = union of that node's child boxes).  Missing / empty children get the neutral box (+inf, -inf).
__global__ void node_kernel(const float4* __restrict__ pts, const float4* __restrict__ child_nodes, int n_child, int n_nodes, float4* __restrict__ nodes) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  const int j = g / FANOUT, c = g % FANOUT;
  if (j >= n_nodes) return;
  float l0 = INFINITY, l1 = INFINITY, l2 = INFINITY, h0 = -INFINITY, h1 = -INFINITY, h2 = -INFINITY;
  const int ci = j * FANOUT + c;
  if (ci < n_child) {
    if (child_nodes == nullptr) {
      for (int k = 0; k < BUCKET; k++) {
        const float4 p = pts[ci * BUCKET + k];
        if (p.x < INFINITY) { l0 = fminf(l0, p.x); l1 = fminf(l1, p.y); l2 = fminf(l2, p.z); h0 = fmaxf(h0, p.x); h1 = fmaxf(h1, p.y); h2 = fmaxf(h2, p.z); }
      }
    } else {
      const float4* r = child_nodes + (size_t)ci * NODE_F4;
      for (int k = 0; k < FANOUT; k++) {
        const float4 a = r[2 * k], b = r[2 * k + 1];
        l0 = fminf(l0, a.x); l1 = fminf(l1, a.y); l2 = fminf(l2, a.z); h0 = fmaxf(h0, b.x); h1 = fmaxf(h1, b.y); h2 = fmaxf(h2, b.z);
      }
    }
  }
  float4* o = nodes + (size_t)j * NODE_F4;
  o[2 * c] = make_float4(l0, l1, l2, 0.f); o[2 * c + 1] = make_float4(h0, h1, h2, 0.f);
}
__global__ void bbox_publish_kernel(const int* __restrict__ bbox, float* __restrict__ out6) {   // decoded box for the query-sort kernel
  if (threadIdx.x < 6) out6[threadIdx.x] = ll_ord2f(bbox[threadIdx.x]);
}

// The index of n_src points: its shape (key width, level sizes), the scratch of its build and its storage.
struct TreeLayout {
  int n_src, bits, sort_bits, n_pad, n_levels = 0, level_count[LL_MAX_LEVELS] = {0};
  bool k32, too_deep = false;
  size_t temp_bytes = 0, node_total = 0;
  int* bbox; void* k0; void* k1; int* v0; int* v1; char* tmp;       // scratch
  float4* pts; float4* nodes; float4* src; float* d_bbox;           // storage
  explicit TreeLayout(int n) : n_src(n) {
    // key width: lidar maps are surfaces, so a grid of 2^b cells per axis has ~4^b occupied cells; b = ceil(log2(n) / 2) - 1 keeps the occupied
    // cells well below a bucket's 32 points (5M points: b = 11, 34 sorted bits = 5 radix passes instead of 8; 30k points: b = 7, 3 passes)
    int lg = 0; while ((1ll << lg) < (long long)(n_src > 0 ? n_src : 1)) lg++;
    bits = (lg + 1) / 2 - 1; if (bits < 5) bits = 5; if (bits > 21) bits = 21;
    sort_bits = 3 * bits + 1;   // one more bit than the key: non-finite points get the key 2^(3 bits) and sort behind every real one
    k32 = sort_bits <= 32;
    if (k32) cub::DeviceRadixSort::SortPairs(nullptr, temp_bytes, (unsigned*)nullptr, (unsigned*)nullptr, (int*)nullptr, (int*)nullptr, n_src > 0 ? n_src : 1, 0, sort_bits);
    else cub::DeviceRadixSort::SortPairs(nullptr, temp_bytes, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int*)nullptr, (int*)nullptr, n_src > 0 ? n_src : 1, 0, sort_bits);
    n_pad = ll_div_up(n_src > 0 ? n_src : 1, BUCKET) * BUCKET;
    // level sizes: level 0 nodes have buckets as children; the top level has exactly one node
    int cnt = ll_div_up(n_pad / BUCKET, FANOUT);
    for (;;) { level_count[n_levels++] = cnt; if (cnt <= 1) break; if (n_levels == LL_MAX_LEVELS) { too_deep = true; break; } cnt = ll_div_up(cnt, FANOUT); }
    for (int l = 0; l < n_levels; l++) node_total += (size_t)level_count[l];
  }
  void scratch_layout(Carve& c) {   // bbox (8 ints) | keys | keys_out | vals | vals_out | CUB temp
    const size_t ksz = k32 ? 4 : 8;
    bbox = c.take<int>(16); k0 = c.take<char>(n_src * ksz); k1 = c.take<char>(n_src * ksz); v0 = c.take<int>(n_src); v1 = c.take<int>(n_src); tmp = c.take<char>(temp_bytes);
  }
  void storage_layout(Carve& c) {   // points | nodes (top level first) | source copy | box
    pts = c.take<float4>(n_pad); nodes = c.take<float4>(node_total * NODE_F4); src = c.take<float4>(n_src); d_bbox = c.take<float>(6);
  }
};
size_t tree_scratch_bytes(int n_src) { TreeLayout L(n_src); return layout_bytes([&](Carve& c) { L.scratch_layout(c); }); }
size_t tree_storage_bytes(int n_src) { TreeLayout L(n_src); return layout_bytes([&](Carve& c) { L.storage_layout(c); }); }

// Enqueued on stream s with its own scratch arena (the corner and the surface index of one map are built side by side: every kernel of a
// 100k-point build is far too small to fill the GPU).  Nothing is read back: the layout is sized from n_src (the non-finite points -- there are
// usually none -- only leave a few all-pad buckets with neutral boxes at the end), the count of finite points and the box stay on the device.
int build_bucket_tree(ll_ctx* ctx, cudaStream_t s, DevBuf& scratch, const float4* d_src, int n_src, BucketTree* t) {
  { DevBuf keep = t->storage; *t = BucketTree(); t->storage = keep; }   // re-indexing in place (ll_map_rebuild) reuses the allocation
  t->n_src = n_src;
  TreeLayout L(n_src);
  if (L.too_deep) { ctx->set_error("map too large for LL_MAX_LEVELS"); return LL_ERR_CAPACITY; }
  LL_CUDA(ctx, scratch.carve([&](Carve& c) { L.scratch_layout(c); }));
  LL_CUDA(ctx, t->storage.carve([&](Carve& c) { L.storage_layout(c); }));
  t->n = n_src; t->n_pad = L.n_pad; t->n_levels = L.n_levels;
  for (int l = 0; l < L.n_levels; l++) t->level_count[l] = L.level_count[l];
  { size_t off = 0; for (int l = t->n_levels - 1; l >= 0; l--) { t->lo[l] = L.nodes + off * NODE_F4; off += (size_t)t->level_count[l]; } }
  t->pts = L.pts; t->src = L.src; t->d_bbox = L.d_bbox;
  int* bbox = L.bbox; int* v0 = L.v0; int* v1 = L.v1;
  bbox_init_kernel<<<1, 32, 0, s>>>(bbox); ctx->launches++;
  if (n_src > 0) {
    int grid = min(ll_div_up(n_src, 256), ctx->num_sms * 8);
    bbox_kernel<<<grid, 256, 0, s>>>(d_src, n_src, bbox); ctx->launches++;
    if (L.k32) {
      unsigned* k0 = (unsigned*)L.k0; unsigned* k1 = (unsigned*)L.k1;
      hilbert_kernel<unsigned><<<ll_div_up(n_src, 256), 256, 0, s>>>(d_src, n_src, bbox, L.bits, k0, v0); ctx->launches++;
      LL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(L.tmp, L.temp_bytes, k0, k1, v0, v1, n_src, 0, L.sort_bits, s));
    } else {
      unsigned long long* k0 = (unsigned long long*)L.k0; unsigned long long* k1 = (unsigned long long*)L.k1;
      hilbert_kernel<unsigned long long><<<ll_div_up(n_src, 256), 256, 0, s>>>(d_src, n_src, bbox, L.bits, k0, v0); ctx->launches++;
      LL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(L.tmp, L.temp_bytes, k0, k1, v0, v1, n_src, 0, L.sort_bits, s));
    }
    ctx->launches += 3 + (L.sort_bits + 7) / 8;
    LL_CUDA(ctx, cudaMemcpyAsync(t->src, d_src, (size_t)n_src * 16, cudaMemcpyDeviceToDevice, s));
  }
  bbox_publish_kernel<<<1, 32, 0, s>>>(bbox, t->d_bbox); ctx->launches++;
  gather_kernel<<<ll_div_up(t->n_pad, 256), 256, 0, s>>>(d_src, v1, bbox, t->n_pad, t->pts); ctx->launches++;
  for (int l = 0; l < t->n_levels; l++) {
    const int n_child = l == 0 ? t->n_pad / BUCKET : t->level_count[l - 1];
    node_kernel<<<ll_div_up(t->level_count[l] * FANOUT, 128), 128, 0, s>>>(t->pts, l == 0 ? nullptr : t->lo[l - 1], n_child, t->level_count[l], t->lo[l]); ctx->launches++;
  }
  LL_CUDA(ctx, cudaGetLastError());
  return LL_OK;
}

TreeView make_view(const BucketTree& t) {
  TreeView v; v.pts = t.pts; v.src = t.src; v.n = t.n; v.n_levels = t.n_levels;
  for (int l = 0; l < LL_MAX_LEVELS; l++) v.nodes[l] = t.lo[l];
  v.bbox = t.d_bbox;
  return v;
}

// ------------------------------------------------------------------------------------------------ search
// One warp per query.  Depth-first over the 32-ary box tree, nearest child first at every node: for the node being expanded at level l, lane c
// holds the lower bound of child c (registers -> a 128-byte row of shared memory per level), a 32-bit mask says which children are still to
// be visited, and "pick" = one REDUX.MIN over the bounds of the remaining children that can still beat the current 5th distance.  The bound is
// tested when a child is PICKED, against the distance list as it is then -- nothing stale is ever expanded, and once the nearest remaining
// child of a node fails the test the whole node is finished.  A bucket = 32 points, one per lane (one coalesced 512-byte load).
// The 5 best (d2, index) pairs live in lanes 0..4, sorted; an insertion is a ballot + two SHFL.UP.  Exact: a box gives a true lower bound of the
// fp32 distance, (d2, index) is a total order, and ties on d2 keep the smaller index, so the result does not depend on the visiting order.
#define KNN_THREADS 256
#define WARPS_PER_CTA (KNN_THREADS / 32)
#define KNN_LEVELS LL_MAX_LEVELS   // 32^8 buckets: more than any map that fits the HBM

__device__ __forceinline__ bool lex_less(float d, int id, float d2, int id2) { return d < d2 || (d == d2 && id < id2); }

// FLANN L2_Simple<float>: result += diff*diff, x then y then z, float accumulation, no contraction.
__device__ __forceinline__ float dist2_exact(float qx, float qy, float qz, float px, float py, float pz) {
  float dx = __fsub_rn(qx, px), dy = __fsub_rn(qy, py), dz = __fsub_rn(qz, pz);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}
// Lower bound of dist2_exact over every point inside the box: same operation sequence on the per-axis gaps, and
// round-to-nearest is monotone, so lb <= d2 holds bit-wise (the search stays exact).
__device__ __forceinline__ float box_lb(float lox, float loy, float loz, float hix, float hiy, float hiz, float qx, float qy, float qz) {
  float ex = fmaxf(fmaxf(__fsub_rn(lox, qx), __fsub_rn(qx, hix)), 0.f);
  float ey = fmaxf(fmaxf(__fsub_rn(loy, qy), __fsub_rn(qy, hiy)), 0.f);
  float ez = fmaxf(fmaxf(__fsub_rn(loz, qz), __fsub_rn(qz, hiz)), 0.f);
  return __fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(ez, ez));
}

// The query's 5 best so far: lane j < 5 holds the j-th smallest (d, id); d5 / id5 = lane 4's entry, known to every lane.
struct LaneTop { float d; int id; float d5; int id5; };
__device__ __forceinline__ void top_init(LaneTop& t) { t.d = INFINITY; t.id = 0x7fffffff; t.d5 = INFINITY; t.id5 = 0x7fffffff; }
// (md, mi) is warp-uniform and lex-less than the 5th entry.  An index that is already in the list is ignored (seeds are real points of the map).
__device__ __forceinline__ void top_insert(LaneTop& t, float md, int mi, int lane) {
  const bool mine = lane < LL_KNN;
  if (__ballot_sync(FULL, mine && t.id == mi)) return;
  const int pos = __popc(__ballot_sync(FULL, mine && !lex_less(md, mi, t.d, t.id)));   // entries that stay in front of the newcomer
  const float ud = __shfl_up_sync(FULL, t.d, 1); const int ui = __shfl_up_sync(FULL, t.id, 1);
  if (mine && lane >= pos) { t.d = lane == pos ? md : ud; t.id = lane == pos ? mi : ui; }
  t.d5 = __shfl_sync(FULL, t.d, LL_KNN - 1); t.id5 = __shfl_sync(FULL, t.id, LL_KNN - 1);
}
// Merge this step's candidates (one per lane, flag c): repeatedly take the smallest one that still beats the 5th entry (<= 5 rounds).
__device__ __forceinline__ void top_merge(LaneTop& t, float d, int id, bool c, int lane) {
  c = c && lex_less(d, id, t.d5, t.id5);   // NaN and +inf distances fail here
  while (__any_sync(FULL, c)) {
    const unsigned key = c ? __float_as_uint(d) : 0xffffffffu;   // non-negative floats order like their bit patterns
    const unsigned mn = __reduce_min_sync(FULL, key);
    const int mi = (int)__reduce_min_sync(FULL, (c && key == mn) ? (unsigned)id : 0x7fffffffu);
    top_insert(t, __uint_as_float(mn), mi, lane);
    if (id == mi && key == mn) c = false;
    c = c && lex_less(d, id, t.d5, t.id5);
  }
}

struct WarpWalk { float lb[KNN_LEVELS][32]; };   // per warp: the child bounds of the node open at every level

// All 32 lanes of the warp call this together; `active` is warp-uniform.
// seed_ids: the query's 5 neighbours of the previous ICP iteration (or null / -1): their distances to the moved query seed the list, so the
// bound is tight before the first box is opened.
__device__ __forceinline__ void warp_knn5(const TreeView& tv, WarpWalk& ws, bool active, float qx, float qy, float qz, LaneTop& t, const int* seed_ids) {
  const int lane = threadIdx.x & 31;
  top_init(t);
  if (!(active && tv.n > 0)) return;
  if (seed_ids) {
    int sid = -1;
    if (lane < LL_KNN) sid = seed_ids[lane];
    if (__any_sync(FULL, sid >= 0)) {
      float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
      if (sid >= 0) p = __ldg(tv.src + sid);
      top_merge(t, sid >= 0 ? dist2_exact(qx, qy, qz, p.x, p.y, p.z) : INFINITY, sid, sid >= 0, lane);
    }
  }
  const int top = tv.n_levels - 1;
  int l = top, idx = 0;          // the node open at level l is node `idx` of that level
  unsigned remv = 0;             // lane k keeps the mask of the children still to visit of the node open at level k
  bool open_node = true;
  for (;;) {
    if (open_node) {             // expand node idx of level l: one box per lane (2 x 16-byte loads, 1 KB per node)
      const float4* r = tv.nodes[l] + (size_t)idx * NODE_F4 + 2 * lane;
      const float4 A = __ldg(r), B = __ldg(r + 1);
      const float lb = box_lb(A.x, A.y, A.z, B.x, B.y, B.z, qx, qy, qz);   // a missing child has the neutral box (+inf, -inf): lb = +inf
      ws.lb[l][lane] = lb;
      const unsigned m = __ballot_sync(FULL, lb <= t.d5 && lb < INFINITY);
      if (lane == l) remv = m;
      open_node = false;   // (every lane only ever reads back its own slot of the row: no synchronisation needed)
    }
    // pick the nearest remaining child of the node open at level l that can still hold a neighbour
    const float lb = ws.lb[l][lane];
    const unsigned rem = __shfl_sync(FULL, remv, l);
    const bool ok = ((rem >> lane) & 1u) && lb <= t.d5;
    const unsigned key = ok ? __float_as_uint(lb) : 0xffffffffu;
    const unsigned mn = __reduce_min_sync(FULL, key);
    if (mn == 0xffffffffu) {     // nothing left here: back to the parent (whose bounds are still in its row)
      if (l == top) break;
      l++; idx >>= 5; continue;
    }
    const unsigned who = __ballot_sync(FULL, key == mn);
    const int c = __ffs(who) - 1;
    const unsigned okm = __ballot_sync(FULL, ok);
    if (lane == l) remv = okm & ~(1u << c);   // (okm is a subset of rem) the children that failed the test now can never pass it later
    const int child = idx * FANOUT + c;
    if (l == 0) {                // a bucket: one point per lane
      const float4 P = __ldg(tv.pts + (size_t)child * BUCKET + lane);
      top_merge(t, dist2_exact(qx, qy, qz, P.x, P.y, P.z), __float_as_int(P.w), true, lane);   // pad points are +inf: never candidates
    } else { l--; idx = child; open_node = true; }
  }
}

// Parity hook (ll_knn): world-frame queries in caller order.
__global__ void __launch_bounds__(KNN_THREADS) knn_query_kernel(TreeView tv, const float4* __restrict__ q, int nq, int* __restrict__ idx5, float* __restrict__ d5) {
  __shared__ WarpWalk walks[WARPS_PER_CTA];
  const int g = blockIdx.x * WARPS_PER_CTA + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const bool have = g < nq;
  float4 p = make_float4(0.f, 0.f, 0.f, 0.f); if (have) p = __ldg(&q[g]);
  const bool active = have && isfinite(p.x) && isfinite(p.y) && isfinite(p.z);
  LaneTop t;
  warp_knn5(tv, walks[threadIdx.x >> 5], active, p.x, p.y, p.z, t, nullptr);
  if (have && lane < LL_KNN) { idx5[g * LL_KNN + lane] = (t.id == 0x7fffffff) ? -1 : t.id; d5[g * LL_KNN + lane] = t.d; }
}

// Spatial sort key of a feature at the current pose: class bit (corner/surface) | 21-bit Hilbert index (7 bits per axis) inside the tree's box.
// Neighbouring queries then sit in the same warp / CTA, walk the same tree nodes and buckets, and hit them in L1.
__global__ void query_key_kernel(KnnBlocksArgs a, unsigned* __restrict__ keys, int* __restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int M = a.n_corner + a.n_surf;
  if (i >= M) return;
  const bool is_corner = i < a.n_corner;
  const float4 f = __ldg(&a.feat[i]);
  double wx, wy, wz; qrot_d(a.pose, (double)f.x, (double)f.y, (double)f.z, wx, wy, wz);
  const float c[3] = {(float)(wx + a.pose[4]), (float)(wy + a.pose[5]), (float)(wz + a.pose[6])};
  const float* bb = is_corner ? a.corner.bbox : a.surf.bbox;   // device memory: the box never visits the host
  // 7 bits per axis: 21-bit curve + class bit = 3 radix passes, and tiles of ~0.3 m are fine enough; non-finite features sort last in their class
  const unsigned h = (isfinite(c[0]) && isfinite(c[1]) && isfinite(c[2])) ? (unsigned)hilbert_key(c, bb, bb + 3, 7) : 0x1fffffu;
  keys[i] = (is_corner ? 0u : 0x200000u) | h; vals[i] = i;
}

// Gates + functor constructors (K7) for one feature whose 5 nearest neighbours are id[0..4] (d4 = the 5th squared distance); lane 0 writes slot `w`.
__device__ __forceinline__ void emit_block(const KnnBlocksArgs& a, const TreeView& tv, bool is_corner, bool active, int w, int id0, int id1, int id2, int id4, float d4) {
  int type = 0; double ax = 0, ay = 0, az = 0, vx = 0, vy = 0, vz = 0;
  if (active) {
    const bool found5 = id4 != 0x7fffffff;
    if (is_corner) {
      if (found5 && (double)d4 < a.max_dis_line) {
        if (a.icp_line) {
          const float4 p1 = __ldg(&tv.src[id0]), p2 = __ldg(&tv.src[id1]);
          double d0 = (double)p1.x - (double)p2.x, d1 = (double)p1.y - (double)p2.y, d2 = (double)p1.z - (double)p2.z;
          double dn = sqrt(d0 * d0 + d1 * d1 + d2 * d2);
          if (!(dn < 0.0001)) {
            // ceres_icp_point2line ctor: unit_vec_ab = (b - a) / |b - a|
            double u0 = (double)p2.x - (double)p1.x, u1 = (double)p2.y - (double)p1.y, u2 = (double)p2.z - (double)p1.z;
            double n = sqrt(u0 * u0 + u1 * u1 + u2 * u2);
            vx = u0 / n; vy = u1 / n; vz = u2 / n; ax = p1.x; ay = p1.y; az = p1.z; type = 1;
            atomicAdd(a.corner_avail, 1);
          }
        }
      }
    } else {
      if (found5 && (double)d4 < a.max_dis_plane) {
        if (a.icp_plane) {
          const float4 pa = __ldg(&tv.src[id0]), pb = __ldg(&tv.src[id2]), pc = __ldg(&tv.src[id4]);
          double b0 = (double)pb.x - (double)pa.x, b1 = (double)pb.y - (double)pa.y, b2 = (double)pb.z - (double)pa.z;
          double nb = sqrt(b0 * b0 + b1 * b1 + b2 * b2); b0 = b0 / nb; b1 = b1 / nb; b2 = b2 / nb;
          double c0 = (double)pc.x - (double)pa.x, c1 = (double)pc.y - (double)pa.y, c2 = (double)pc.z - (double)pa.z;
          double nc = sqrt(c0 * c0 + c1 * c1 + c2 * c2); c0 = c0 / nc; c1 = c1 / nc; c2 = c2 / nc;
          vx = b1 * c2 - b2 * c1; vy = b2 * c0 - b0 * c2; vz = b0 * c1 - b1 * c0;   // NOT re-normalised (ceres_icp.hpp:334)
          ax = pa.x; ay = pa.y; az = pa.z; type = 2;
        }
        atomicAdd(a.surf_avail, 1);
      }
    }
  }
  if (type != 0) atomicAdd(a.n_blocks, 1);   // residual_block_ids.size() of this ICP iteration (the cap's drop rule needs it, :436)
  a.blk_a[w] = make_float4((float)ax, (float)ay, (float)az, __int_as_float(type));
  a.blk_v[(size_t)w * 3 + 0] = vx; a.blk_v[(size_t)w * 3 + 1] = vy; a.blk_v[(size_t)w * 3 + 2] = vz;
}

// K6 + K7 fused, one warp per scan feature, features taken in spatially sorted order (perm).
// Writes one residual-block slot per feature (indexed by the ORIGINAL feature order): blk_a[slot] = (a.x, a.y, a.z, type) with
// type 0 invalid / 1 line / 2 plane, blk_v[slot*3..] = unit line direction or (un-normalised) plane normal, in fp64.
__global__ void __launch_bounds__(KNN_THREADS) knn_blocks_kernel(KnnBlocksArgs a) {
  if (a.st->icp_done) return;   // launched ahead of the termination test by the host: the ICP loop has already ended
  __shared__ WarpWalk walks[WARPS_PER_CTA];
  const int j = blockIdx.x * WARPS_PER_CTA + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int M = a.n_corner + a.n_surf;
  const bool have = j < M;
  const int w = have ? (a.perm ? a.perm[j] : j) : 0;      // original feature index
  const bool is_corner = w < a.n_corner;
  const TreeView& tv = is_corner ? a.corner : a.surf;
  float4 f = make_float4(0.f, 0.f, 0.f, 0.f); if (have) f = __ldg(&a.feat[w]);
  // pointAssociateToMap (non-deblur branch): p_w = q_curr * p + t_curr in fp64, stored as fp32
  const double* qc = a.pose; const double* tc = a.pose + 4;
  double wx, wy, wz; qrot_d(qc, (double)f.x, (double)f.y, (double)f.z, wx, wy, wz);
  float qx = (float)(wx + tc[0]), qy = (float)(wy + tc[1]), qz = (float)(wz + tc[2]);
  if (a.deblur) {
    // pointAssociateToMap, deblur branch (:627-654, if_undistore_in_matching = 1): Rodrigues-interpolated increment applied before q_last
    const RegDevState* st = a.st;
    const double is = (double)refine_blur_f(f.w, (float)st->min_ts, (float)st->max_ts);
    if (is != 1.0) {
      const double th = st->interp_theta * is; double sn, cs; sincos(th, &sn, &cs); const double oc = 1.0 - cs;
      const double* H = st->interp_hat; const double* H2 = st->interp_hat_sq;
      const double px = (double)f.x, py = (double)f.y, pz = (double)f.z;
      double rx = ((1.0 + sn * H[0] + oc * H2[0]) * px + (sn * H[1] + oc * H2[1]) * py) + (sn * H[2] + oc * H2[2]) * pz;
      double ry = ((sn * H[3] + oc * H2[3]) * px + (1.0 + sn * H[4] + oc * H2[4]) * py) + (sn * H[5] + oc * H2[5]) * pz;
      double rz = ((sn * H[6] + oc * H2[6]) * px + (sn * H[7] + oc * H2[7]) * py) + (1.0 + sn * H[8] + oc * H2[8]) * pz;
      rx += st->x[4] * (is * 1.0); ry += st->x[5] * (is * 1.0); rz += st->x[6] * (is * 1.0);
      double ox, oy, oz; qrot_d(st->pose_last, rx, ry, rz, ox, oy, oz);
      qx = (float)(ox + st->pose_last[4]); qy = (float)(oy + st->pose_last[5]); qz = (float)(oz + st->pose_last[6]);
    }
  }
  // Non-finite features: the corner loop skips them explicitly (:242-245); the surface loop does not (:347-351), but a NaN query makes every
  // squared distance NaN and `NaN < 50.0` (:353) rejects the match, so the block set is the same.
  const bool finite_in = isfinite(f.x) && isfinite(f.y) && isfinite(f.z);
  bool owned = true;
  if (a.world > 1) owned = finite_in && __ldg(&a.shard_owner[shard_cell_index(a.grid, qx, qy, qz)]) == a.rank;   // shard.cu: every point of space has exactly one owner
  // Residual-block cap, pre-skip (:232-238 corners, :339-345 surfaces): with N features of this class and N > 2 cap, a feature is skipped when
  // rand * N > 2 cap (float arithmetic, like m_rand_float), before it is transformed or searched.  Drawn per (seed, ICP iteration, class, index).
  bool skipped = false;
  { const int ncls = is_corner ? a.n_corner : a.n_surf;
    if (have && ncls > 2 * a.cap) skipped = ll_cap_uniform_f(a.rng_seed, a.st->icp_iter, is_corner ? 0 : 1, is_corner ? w : w - a.n_corner) * (float)ncls > (float)(2 * a.cap); }
  const bool active = have && owned && finite_in && !skipped;
  LaneTop t;
  warp_knn5(tv, walks[threadIdx.x >> 5], active, qx, qy, qz, t, (a.seed_ids && have) ? a.seed_ids + (size_t)w * LL_KNN : nullptr);
  if (!have) return;
  if (active && lane < LL_KNN) {   // the neighbours seed the next ICP iteration's search (5 lanes, one 20-byte row)
    if (a.seed_ids) a.seed_ids[(size_t)w * LL_KNN + lane] = (t.id == 0x7fffffff) ? -1 : t.id;
    if (a.knn_d) a.knn_d[(size_t)w * LL_KNN + lane] = t.d;
  }
  const int id0 = __shfl_sync(FULL, t.id, 0), id1 = __shfl_sync(FULL, t.id, 1), id2 = __shfl_sync(FULL, t.id, 2);
  if (lane != 0) return;
  emit_block(a, tv, is_corner, active, w, id0, id1, id2, t.id5, t.d5);
}

int launch_knn_query(ll_ctx* ctx, const BucketTree& t, const float4* d_q, int nq, int* d_idx, float* d_d) {
  if (nq == 0) return LL_OK;
  knn_query_kernel<<<ll_div_up(nq, WARPS_PER_CTA), KNN_THREADS, 0, ctx->stream>>>(make_view(t), d_q, nq, d_idx, d_d); ctx->launches++;
  LL_CUDA(ctx, cudaGetLastError());
  return LL_OK;
}
// Sorts the features spatially (once per registration, at the initial pose): perm[] lists corner features then surface features.
// keys | keys_out | vals | CUB temp (the sorted values go to perm)
struct QuerySortLayout {
  size_t tmp_bytes = 0; unsigned* k0; unsigned* k1; int* v0; char* tmp;
  explicit QuerySortLayout(int M) { cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, (unsigned*)nullptr, (unsigned*)nullptr, (int*)nullptr, (int*)nullptr, M, 0, 22); }
  void layout(Carve& c, int M) { k0 = c.take<unsigned>(M); k1 = c.take<unsigned>(M); v0 = c.take<int>(M); tmp = c.take<char>(tmp_bytes); }
};
size_t query_sort_bytes(int M) { QuerySortLayout q(M); return layout_bytes([&](Carve& c) { q.layout(c, M); }); }
int launch_query_sort(ll_ctx* ctx, cudaStream_t s, DevBuf& scratch, const KnnBlocksArgs& a, int* d_perm) {
  const int M = a.n_corner + a.n_surf;
  if (M == 0) return LL_OK;
  QuerySortLayout q(M);
  LL_CUDA(ctx, scratch.carve([&](Carve& c) { q.layout(c, M); }));
  query_key_kernel<<<ll_div_up(M, 256), 256, 0, s>>>(a, q.k0, q.v0);
  LL_CUDA(ctx, cub::DeviceRadixSort::SortPairs(q.tmp, q.tmp_bytes, q.k0, q.k1, q.v0, d_perm, M, 0, 22, s));
  ctx->launches += 4;
  return LL_OK;
}
int launch_knn_blocks(ll_ctx* ctx, const KnnBlocksArgs& a) {
  int M = a.n_corner + a.n_surf;
  if (M == 0) return LL_OK;
  knn_blocks_kernel<<<ll_div_up(M, WARPS_PER_CTA), KNN_THREADS, 0, ctx->stream>>>(a);
  ctx->launches++;
  LL_CUDA(ctx, cudaGetLastError());
  return LL_OK;
}
