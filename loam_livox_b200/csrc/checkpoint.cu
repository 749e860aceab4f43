// What the mapper image and the loop image share (kernels.cuh, "byte images"): the header, the history section and the cell-map section, each
// laid out, written, checked and restored once.  Host code only.
#include <algorithm>
#include <cmath>
#include <cstring>
#include "common.cuh"
#include "kernels.cuh"

size_t image_header(const ImageKind& kind, uint32_t version, const uint64_t* len, void* header) {
  uint8_t* h = (uint8_t*)header;
  const int sections = kind.count(version);
  const uint64_t head = 24 + 16 * (uint64_t)sections;
  memset(h, 0, head);
  memcpy(h, kind.magic, 8); img_put<uint32_t>(h + 8, version); img_put<uint32_t>(h + 12, kind.config_bytes);
  uint64_t off = head;
  for (int k = 0; k < sections; k++) { img_put<uint64_t>(h + 24 + 16 * k, off); img_put<uint64_t>(h + 32 + 16 * k, len[k]); off += len[k]; }
  img_put<uint64_t>(h + 16, off);
  return (size_t)off;
}

int image_structure(const void* image, size_t bytes, const ImageKind& kind, ll_image_section* sec, std::string* err) {
  auto fail = [&](const std::string& msg) { if (err) *err = msg; return LL_ERR_INVALID; };
  const uint8_t* b = (const uint8_t*)image;
  if (!b || bytes < 24 + 16 * (size_t)kind.sections) return fail("shorter than the image header");
  char magic[8]; uint32_t version, config_bytes; uint64_t total;
  memcpy(magic, b, 8); memcpy(&version, b + 8, 4); memcpy(&config_bytes, b + 12, 4); memcpy(&total, b + 16, 8);
  if (memcmp(magic, kind.magic, 8) != 0) return fail(std::string("not a ") + kind.name + " image (magic)");
  if (version < kind.version || version > kind.max_version) return fail("unknown image version");
  const int sections = kind.count(version);
  const size_t head = 24 + 16 * (size_t)sections;
  if (bytes < head) return fail("shorter than the image header");
  memcpy(sec, b + 24, 16 * (size_t)sections);
  if (config_bytes != kind.config_bytes) return fail(std::string("config size differs from this library's ") + kind.config_name);
  if (total != bytes) return fail("image size differs from the header's total_bytes");
  // every section inside the image after the header, no two overlapping
  std::vector<int> order(sections);
  for (int k = 0; k < sections; k++) {
    const ll_image_section& s = sec[k];
    if (s.offset < head || s.offset > bytes || s.length > bytes - s.offset) return fail("section outside the image");
    order[k] = k;
  }
  std::sort(order.begin(), order.end(), [&](int a, int c) {
    const ll_image_section &x = sec[a], &y = sec[c];
    return x.offset != y.offset ? x.offset < y.offset : x.length < y.length;
  });
  for (int k = 1; k < sections; k++) {
    const ll_image_section &p = sec[order[k - 1]], &q = sec[order[k]];
    if (p.offset + p.length > q.offset) return fail("overlapping sections");
  }
  return LL_OK;
}

bool finite_xyz(const uint8_t* p) { float v[3]; memcpy(v, p, 12); return std::isfinite(v[0]) && std::isfinite(v[1]) && std::isfinite(v[2]); }
bool finite_d(const double* d, int n) { for (int k = 0; k < n; k++) if (!std::isfinite(d[k])) return false; return true; }

// ---------------------------------------------------------------------------------------------- history section
uint64_t history_bytes(const HistoryWindow& w) { return HIS_HEAD + 4 * (uint64_t)w.segs.size() + 16 * (uint64_t)w.live(); }

int history_write(ll_ctx* ctx, const HistoryWindow& w, uint8_t* p) {
  const size_t live = w.live();
  img_put<int64_t>(p, (int64_t)w.segs.size()); img_put<int64_t>(p + 8, (int64_t)live); p += HIS_HEAD;
  for (const auto& sg : w.segs) { img_put<int32_t>(p, (int32_t)sg.second); p += 4; }
  if (live) LL_CUDA(ctx, cudaMemcpyAsync(p, w.data(), live * 16, cudaMemcpyDeviceToHost, ctx->stream));
  return LL_OK;
}

const char* history_section(const uint8_t* p, uint64_t L, bool finite, HistoryView* v) {
  if (L < HIS_HEAD) return "history section shorter than its counts";
  const int64_t ns = img_get<int64_t>(p), np = img_get<int64_t>(p + 8);
  if (ns < 0 || np < 0 || (uint64_t)ns > (L - HIS_HEAD) / 4 || (uint64_t)np > (L - HIS_HEAD) / 16 || HIS_HEAD + 4 * (uint64_t)ns + 16 * (uint64_t)np != L)
    return "history counts disagree with the section length";
  int64_t sum = 0;
  for (int64_t k = 0; k < ns; k++) { const int32_t z = img_get<int32_t>(p + HIS_HEAD + 4 * k); if (z < 0) return "negative history segment size"; sum += z; }
  if (sum != np) return "history segment sizes do not sum to its points";
  const uint8_t* q = p + HIS_HEAD + 4 * ns;
  if (finite) for (int64_t k = 0; k < np; k++) if (!finite_xyz(q + 16 * k)) return "non-finite history point";
  v->n_seg = ns; v->n_pts = np; v->sizes = p + HIS_HEAD; v->pts = q;
  return nullptr;
}

int history_restore(ll_ctx* ctx, HistoryWindow& w, const HistoryView& v) {
  cudaStream_t s = ctx->stream;
  float4* d = nullptr;
  if (v.n_pts) {
    LL_CUDA(ctx, ctx->scratch.carve([&](Carve& k) { d = k.take<float4>((size_t)v.n_pts); }));
    LL_CUDA(ctx, cudaMemcpyAsync(d, v.pts, (size_t)v.n_pts * 16, cudaMemcpyHostToDevice, s));
  }
  size_t off = 0;
  for (int64_t k = 0; k < v.n_seg; k++) {
    const size_t n = (size_t)img_get<int32_t>(v.sizes + 4 * k);
    LL_TRY(w.push(ctx, d ? d + off : nullptr, n));
    off += n;
  }
  LL_CUDA(ctx, cudaStreamSynchronize(s));   // (the scratch upload may be reallocated by the next carve)
  return LL_OK;
}

// ---------------------------------------------------------------------------------------------- cell-map section
uint64_t cells_bytes(const CellsView& n, bool incarnations) { return CELLS_HEAD + (incarnations ? 20 : 16) * (uint64_t)(n.n_cells + n.n_pts); }

int cells_write(ll_ctx* ctx, ll_cellmap* m, const CellsView& n, uint8_t* p, const CmHeld* held) {
  img_put<int32_t>(p, n.frame_idx); img_put<int32_t>(p + 4, n.n_oor); img_put<int64_t>(p + 8, n.n_cells); img_put<int64_t>(p + 16, n.n_pts);
  return cm_export(ctx, m, (int)n.n_cells, (int)n.n_pts, p + CELLS_HEAD, held);
}

const char* cells_section(const uint8_t* p, uint64_t L, bool incarnations, CellsView* v) {
  const uint64_t rec = incarnations ? 20 : 16;   // bytes per cell and per point
  if (L < CELLS_HEAD) return "cell-map section shorter than its counts";
  const int32_t fi = img_get<int32_t>(p), oor = img_get<int32_t>(p + 4);
  const int64_t nc = img_get<int64_t>(p + 8), np = img_get<int64_t>(p + 16);
  if (nc < 0 || np < 0 || (uint64_t)nc > (L - CELLS_HEAD) / rec || (uint64_t)np > (L - CELLS_HEAD) / rec || CELLS_HEAD + rec * (uint64_t)(nc + np) != L)
    return "cell-map counts disagree with the section length";
  if (fi < 0 || oor < 0) return "cell-map frame index or out-of-range count negative";
  const uint8_t* cells = p + CELLS_HEAD; const uint8_t* pts = cells + 16 * nc;
  const uint8_t* cur = incarnations ? pts + 16 * np : nullptr; const uint8_t* ord = incarnations ? cur + 4 * nc : nullptr;
  uint64_t prev = 0;
  for (int64_t k = 0; k < nc; k++) {
    const ll_image_cell e = img_get<ll_image_cell>(cells + 16 * k);
    if (e.key >> 63) return "cell key with bit 63 set";
    if (k > 0 && e.key <= prev) return "cell keys not strictly ascending";
    if (e.create_frame < 0 || e.create_frame > fi || e.last_update < 0 || e.last_update > fi) return "cell stamp outside 0 ... current_frame_idx";
    if (incarnations) {
      const int32_t c = img_get<int32_t>(cur + 4 * k);
      if (c < 0 || c > fi) return "incarnation ordinal outside 0 ... current_frame_idx";   // one revisit per cell and append at most
      v->max_cur = std::max(v->max_cur, c);
    }
    prev = e.key;
  }
  for (int64_t k = 0; k < np; k++) {
    const ll_image_cell_point q = img_get<ll_image_cell_point>(pts + 16 * k);
    if (!(std::isfinite(q.x) && std::isfinite(q.y) && std::isfinite(q.z))) return "non-finite cell-map point";
    if (q.cell < 0 || q.cell >= nc) return "cell-map point's cell rank >= the cell count";
    if (incarnations) {
      const int32_t o = img_get<int32_t>(ord + 4 * k), c = img_get<int32_t>(cur + 4 * q.cell);
      if (o < 0 || o > c) return "cell-map point's incarnation outside 0 ... its cell's current one";
      v->replaced += o != c;
    }
  }
  v->frame_idx = fi; v->n_oor = oor; v->n_cells = nc; v->n_pts = np; v->rec = cells;
  if (incarnations) v->cur = cur;
  return nullptr;
}

int cells_restore(ll_ctx* ctx, ll_cellmap* m, const CellsView& v, bool incarnations, int* slot_of_rank) {
  return cm_import(ctx, m, v.frame_idx, v.n_oor, v.rec, (int)v.n_cells, (int)v.n_pts, incarnations, slot_of_rank);
}

const char* load_capacity(const CellsView& c, const HistoryView& h, const int* max_cells) {
  // ll_cellmap_append does not return from a full table: the import must never make one
  if (max_cells && c.n_cells > table_capacity(*max_cells) / 2) return "cell table more than half full: load with a larger max_cells";
  if (c.n_pts > ((int64_t)1 << 30) || h.n_pts > INT32_MAX) return "more points than a map holds";
  return nullptr;
}
