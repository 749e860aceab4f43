// The cell map's state and cell key, shared by cellmap.cu (the map) and keyframe.cu (keyframes over its cells).
#pragma once
#include "common.cuh"

#define CM_EMPTY 0xffffffffffffffffull
#define CM_BIAS (1 << 20)             // cell indices -2^20 ... 2^20 - 1 fit the 21-bit fields of a key; an append rejects points beyond them

struct ll_cellmap {
  int device = 0;
  float resolution = 0.5f;          // what set_resolution(r) stores: r / 2
  int revisit_threshold = 2147483647;
  int current_frame_idx = 0;
  int n_pts = 0, cap_pts = 0;       // used / allocated entries of the point store (dead points included until the next rebuild)
  int n_cells = 0;                  // cells after the last append (the first append into an empty map is set_point_cloud)
  int n_out_of_range = 0;           // points rejected so far for a cell index beyond the key's range
  int table_cap = 0;                // power of two
  int generation = 0;               // bumped when the store is rebuilt or re-imported: slot / epoch references held outside (keyframes) are void
  unsigned long long* keys = nullptr; int* last_update = nullptr; int* create_frame = nullptr; int* epoch = nullptr; int* bump = nullptr;
  int* d_counters = nullptr;        // [0] number of cells, [1] scratch
  float4* pts = nullptr; int* pt_slot = nullptr; int* pt_epoch = nullptr;
  DevBuf table_buf, store_buf, store_alt, out_buf, tmp_buf;
};

__device__ __forceinline__ unsigned long long cm_pack(int k, int j, int i) {
  return ((unsigned long long)(unsigned)(k + CM_BIAS) << 42) | ((unsigned long long)(unsigned)(j + CM_BIAS) << 21) | (unsigned long long)(unsigned)(i + CM_BIAS);
}
__device__ __forceinline__ void cm_unpack(unsigned long long key, int& k, int& j, int& i) {
  k = (int)((key >> 42) & 0x1fffffull) - CM_BIAS; j = (int)((key >> 21) & 0x1fffffull) - CM_BIAS; i = (int)(key & 0x1fffffull) - CM_BIAS;
}

// The loop image (ll_mapper_loop_save) keeps, beside a cell's current incarnation, those the open keyframes hold: `held`, their sorted, distinct
// (slot << 32 | epoch) ids.  A kept incarnation leaves as its ordinal: 0 for the cell's first incarnation (epoch 0, the one ll_keyframe_analyze
// builds incrementally), otherwise 1 + the held incarnations of the slot with 0 < epoch < e.  Ordinals keep the epoch order of every cell.
__host__ __device__ inline int cm_lower_bound(const unsigned long long* a, int n, unsigned long long x) {
  int lo = 0, hi = n;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (a[mid] < x) lo = mid + 1; else hi = mid; }
  return lo;
}
__host__ __device__ inline int cm_ordinal(const unsigned long long* held, int n_held, int s, int e) {
  if (e == 0) return 0;
  const unsigned long long base = (unsigned long long)(unsigned)s << 32;
  const int lo = cm_lower_bound(held, n_held, base), at = cm_lower_bound(held, n_held, base | (unsigned)e);
  return 1 + (at - lo) - ((lo < n_held && held[lo] == base) ? 1 : 0);
}
