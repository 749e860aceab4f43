// Spatial sharding of the match map across GPUs (BASELINE.json config C4; SURVEY.md 8(e)).
//
// The reference has no multi-GPU path; what it fixes is the pair of match gates that make owner + halo search exact:
//   surface: the 5th squared distance must be < m_maximum_dis_plane_for_match = 50.0  -> halo sqrt(50) = 7.07 m
//   corner : ... < m_maximum_dis_line_for_match = 2.0                                 -> halo sqrt(2)  = 1.42 m
//   (loam_livox/source/point_cloud_registration.hpp:64-65, :254, :353)
// A correspondence whose 5th neighbour lies beyond the gate is rejected anyway, and a shard is a subset of the map (distances can only grow), so
// searching [points of the cells a rank owns] + [every point within the halo of one of those cells] gives, for every ACCEPTED correspondence,
// exactly the neighbours a search of the whole map gives.  Compaction keeps the input order, so index ties break the same way.
//
// Layout: a regular grid of cubic cells (cell_size) over the bounding box of the whole map; cells in Morton order are cut into `world` contiguous
// ranges with (nearly) equal numbers of map points; rank r owns range r.  The border cells extend outwards without bound, so every query has
// exactly one owner, wherever the pose estimate puts it.
#include <cub/cub.cuh>
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>
#include "common.cuh"
#include "kernels.cuh"

__global__ void sh_hist_kernel(const float4* __restrict__ p, int n, ShardGrid g, int* __restrict__ hist) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 q = p[i];
  if (!(isfinite(q.x) && isfinite(q.y) && isfinite(q.z))) return;
  atomicAdd(&hist[shard_cell_index(g, q.x, q.y, q.z)], 1);
}
// keep[i] = 1 when point i belongs to this rank's shard: one of the cells within `halo` of the point is owned by `rank`.
// The distance to a border cell is taken to the cell extended outwards without bound (which, for a point inside the map's box, is the distance to the cell itself).
__global__ void sh_keep_kernel(const float4* __restrict__ p, int n, ShardGrid g, const int* __restrict__ owner, int rank, float halo, unsigned char* __restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 q = p[i];
  unsigned char k = 0;
  if (isfinite(q.x) && isfinite(q.y) && isfinite(q.z)) {
    const float c[3] = {q.x, q.y, q.z}; int lo[3], hi[3];
#pragma unroll
    for (int a = 0; a < 3; a++) {
      lo[a] = max(0, min(g.dims[a] - 1, (int)floorf((c[a] - halo - g.origin[a]) * g.inv_cell)));
      hi[a] = max(0, min(g.dims[a] - 1, (int)floorf((c[a] + halo - g.origin[a]) * g.inv_cell)));
    }
    const float h2 = halo * halo;
    for (int z = lo[2]; z <= hi[2] && !k; z++)
      for (int y = lo[1]; y <= hi[1] && !k; y++)
        for (int x = lo[0]; x <= hi[0]; x++) {
          if (owner[(z * g.dims[1] + y) * g.dims[0] + x] != rank) continue;
          const int ci[3] = {x, y, z}; float d2 = 0.f;
#pragma unroll
          for (int a = 0; a < 3; a++) {
            const float blo = g.origin[a] + (float)ci[a] * g.cell, bhi = blo + g.cell;
            float e = 0.f;
            if (c[a] < blo && ci[a] > 0) e = blo - c[a];                    // cell 0 reaches -inf
            else if (c[a] > bhi && ci[a] < g.dims[a] - 1) e = c[a] - bhi;    // the last cell reaches +inf
            d2 += e * e;
          }
          if (d2 <= h2) { k = 1; break; }
        }
  }
  keep[i] = k;
}

static inline unsigned long long morton3(unsigned x, unsigned y, unsigned z) {
  auto spread = [](unsigned long long v) { v &= 0x1fffffull; v = (v | v << 32) & 0x1f00000000ffffull; v = (v | v << 16) & 0x1f0000ff0000ffull; v = (v | v << 8) & 0x100f00f00f00f00full;
                                           v = (v | v << 4) & 0x10c30c30c30c30c3ull; v = (v | v << 2) & 0x1249249249249249ull; return v; };
  return spread(x) | (spread(y) << 1) | (spread(z) << 2);
}

extern "C" {

// Pure host logic (no GPU): cells in Morton order, cut into `world` contiguous ranges of nearly equal point count; owner_out[cell] = rank.
// A cell goes to rank floor(points_before_it * world / total): every rank's range is contiguous along the curve, empty cells follow their predecessor.
int ll_shard_plan(const int* cell_counts, const int dims[3], int world, int* owner_out) {
  if (!cell_counts || !dims || !owner_out || world < 1 || dims[0] < 1 || dims[1] < 1 || dims[2] < 1) return LL_ERR_INVALID;
  const size_t nc = (size_t)dims[0] * dims[1] * dims[2];
  std::vector<std::pair<unsigned long long, int>> order(nc);
  for (int z = 0; z < dims[2]; z++) for (int y = 0; y < dims[1]; y++) for (int x = 0; x < dims[0]; x++) {
    const int c = (z * dims[1] + y) * dims[0] + x; order[c] = {morton3((unsigned)x, (unsigned)y, (unsigned)z), c};
  }
  std::sort(order.begin(), order.end());
  long long total = 0; for (size_t c = 0; c < nc; c++) total += cell_counts[c];
  long long before = 0;
  for (size_t k = 0; k < nc; k++) {
    const int c = order[k].second;
    int r = total > 0 ? (int)((before * (long long)world) / total) : (int)((k * (size_t)world) / nc);
    if (r > world - 1) r = world - 1;
    owner_out[c] = r; before += cell_counts[c];
  }
  return LL_OK;
}

int ll_map_build_sharded(ll_ctx* ctx, const void* corner, size_t nc, const void* surf, size_t ns, int fmt, int where, int rank, int world, float cell_size,
                         float halo_corner, float halo_surf, ll_map** out) {
  if (!ctx || !out || world < 1 || world > 8 || rank < 0 || rank >= world || !(cell_size > 0.f) || !(halo_corner >= 0.f) || !(halo_surf >= 0.f)) return LL_ERR_INVALID;
  cudaSetDevice(ctx->device);
  cudaStream_t s = ctx->stream;
  *out = nullptr;
  const size_t nmax = nc > ns ? nc : ns;
  size_t sel_bytes = 0;
  cub::DeviceSelect::Flagged(nullptr, sel_bytes, (const float4*)nullptr, (const unsigned char*)nullptr, (float4*)nullptr, (int*)nullptr, (int)(nmax > 0 ? nmax : 1), s);
  // feat_buf: [corner cloud | surface cloud | compacted cloud]; scratch2: bbox, histogram / owner table, keep flags, CUB temp
  float4* d_c; float4* d_s; float4* d_k;
  LL_CUDA(ctx, ctx->feat_buf.carve([&](Carve& c) { d_c = c.take<float4>(nc); d_s = c.take<float4>(ns); d_k = c.take<float4>(nmax); }));
  LL_TRY(upload_cloud(ctx, s, corner, nc, fmt, where, d_c));
  LL_TRY(upload_cloud(ctx, s, surf, ns, fmt, where, d_s));
  // ---- grid over the bounding box of the whole map (identical on every rank: every rank sees the same two clouds)
  int* d_bbox = nullptr;
  LL_CUDA(ctx, ctx->scratch2.carve([&](Carve& c) { d_bbox = c.take<int>(16); }));
  bbox_init_kernel<<<1, 32, 0, s>>>(d_bbox); ctx->launches++;   // (knn.cu; the count of finite points in d_bbox[6] is not used here)
  if (nc) { bbox_kernel<<<std::min(ll_div_up((int)nc, 256), ctx->num_sms * 8), 256, 0, s>>>(d_c, (int)nc, d_bbox); ctx->launches++; }
  if (ns) { bbox_kernel<<<std::min(ll_div_up((int)ns, 256), ctx->num_sms * 8), 256, 0, s>>>(d_s, (int)ns, d_bbox); ctx->launches++; }
  int hb[6];
  LL_CUDA(ctx, cudaMemcpyAsync(hb, d_bbox, sizeof(hb), cudaMemcpyDeviceToHost, s));
  LL_CUDA(ctx, cudaStreamSynchronize(s));
  ll_map* m = new ll_map(); m->device = ctx->device; m->rank = rank; m->world = world; m->cell_size = cell_size; m->halo[0] = halo_corner; m->halo[1] = halo_surf;
  ShardGrid& g = m->grid; g.cell = cell_size; g.inv_cell = 1.0f / cell_size;
  float lo[3], hi[3];
  for (int k = 0; k < 3; k++) { lo[k] = ll_ord2f(hb[k]); hi[k] = ll_ord2f(hb[3 + k]); }
  size_t ncell = 1;
  for (int k = 0; k < 3; k++) {
    if (!(lo[k] <= hi[k])) { lo[k] = 0.f; hi[k] = 0.f; }   // no finite point at all
    g.origin[k] = lo[k];
    g.dims[k] = (int)floorf((hi[k] - lo[k]) * g.inv_cell) + 1;
    ncell *= (size_t)g.dims[k];
  }
  auto fail = [&](int st, const char* why) { if (why) ctx->set_error(why); ll_map_release(m); return st; };
  if (ncell > ((size_t)1 << 24)) return fail(LL_ERR_CAPACITY, "shard grid has more than 2^24 cells: raise cell_size");
  // ---- points per cell -> owner table (host, deterministic) -> device
  int* d_hist; unsigned char* d_keep; int* d_cnt; char* d_tmp;
  auto layout = [&](Carve& c) { d_bbox = c.take<int>(16); d_hist = c.take<int>(ncell); d_keep = c.take<unsigned char>(nmax + 1); d_cnt = c.take<int>(1); d_tmp = c.take<char>(sel_bytes); };
  if (ctx->scratch2.carve(layout) != cudaSuccess) return fail(LL_ERR_CUDA, "shard scratch allocation failed");
  cudaMemsetAsync(d_hist, 0, ncell * 4, s);
  if (nc) { sh_hist_kernel<<<ll_div_up((int)nc, 256), 256, 0, s>>>(d_c, (int)nc, g, d_hist); ctx->launches++; }
  if (ns) { sh_hist_kernel<<<ll_div_up((int)ns, 256), 256, 0, s>>>(d_s, (int)ns, g, d_hist); ctx->launches++; }
  m->h_owner.resize(ncell);
  std::vector<int> hist(ncell);
  if (cudaMemcpyAsync(hist.data(), d_hist, ncell * 4, cudaMemcpyDeviceToHost, s) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess) return fail(LL_ERR_CUDA, "shard histogram read-back failed");
  ll_shard_plan(hist.data(), g.dims, world, m->h_owner.data());
  if (m->shard_owner.reserve(ncell * 4) != cudaSuccess) return fail(LL_ERR_CUDA, "shard owner table allocation failed");
  cudaMemcpyAsync(m->shard_owner.p, m->h_owner.data(), ncell * 4, cudaMemcpyHostToDevice, s);
  // ---- this rank's shard of each cloud: owner cells + halo, compacted in input order, then indexed
  // (1 + 1e-4) h + 1 mm: a superset is always safe, and it absorbs the rounding of the fp32 box arithmetic against the fp32 gate test
  const float4* srcs[2] = {d_c, d_s}; const size_t ns2[2] = {nc, ns}; const float halos[2] = {halo_corner * 1.0001f + 1e-3f, halo_surf * 1.0001f + 1e-3f};
  for (int w = 0; w < 2; w++) {
    int kept = 0;
    if (ns2[w] > 0) {
      sh_keep_kernel<<<ll_div_up((int)ns2[w], 256), 256, 0, s>>>(srcs[w], (int)ns2[w], g, (const int*)m->shard_owner.p, rank, halos[w], d_keep); ctx->launches++;
      if (cub::DeviceSelect::Flagged(d_tmp, sel_bytes, srcs[w], d_keep, d_k, d_cnt, (int)ns2[w], s) != cudaSuccess) return fail(LL_ERR_CUDA, "shard compaction failed");
      ctx->launches += 2;
      if (cudaMemcpyAsync(&kept, d_cnt, 4, cudaMemcpyDeviceToHost, s) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess) return fail(LL_ERR_CUDA, "shard count read-back failed");
    }
    m->shard_total[w] = (long long)ns2[w];
    const int st = build_bucket_tree(ctx, s, ctx->scratch, d_k, kept, &m->tree[w]);
    if (st != LL_OK) return fail(st, nullptr);
  }
  if (cudaStreamSynchronize(s) != cudaSuccess) return fail(LL_ERR_CUDA, "shard build failed");
  *out = m; return LL_OK;
}

// What a caller (or a test) needs to reproduce the ownership on the host: the grid and the owner table.  owner_out may be NULL (query sizes first).
int ll_map_shard_info(const ll_map* map, ll_shard_info* info, int* owner_out, size_t owner_cap) {
  if (!map || !info) return LL_ERR_INVALID;
  memset(info, 0, sizeof(*info));
  info->rank = map->rank; info->world = map->world; info->cell_size = map->grid.cell; info->halo_corner = map->halo[0]; info->halo_surf = map->halo[1];
  for (int k = 0; k < 3; k++) { info->origin[k] = map->grid.origin[k]; info->dims[k] = map->grid.dims[k]; }
  info->kept_corner = (long long)map->tree[0].n_src; info->kept_surf = (long long)map->tree[1].n_src; info->total_corner = map->shard_total[0]; info->total_surf = map->shard_total[1];
  if (owner_out) {
    if (owner_cap < map->h_owner.size()) return LL_ERR_CAPACITY;
    memcpy(owner_out, map->h_owner.data(), map->h_owner.size() * sizeof(int));
  }
  return LL_OK;
}

}  // extern "C"
