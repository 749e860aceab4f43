// K10 building blocks shared by the stand-alone kernels (cloud.cu) and the fused solver kernel (solve.cu):
// compute_inlier_residual_threshold (point_cloud_registration.hpp:153-161) = de-duplicate the per-block L1 norms (std::set<double>), take element
// floor(ratio * size).
#pragma once
#define L1_EMPTY 0xffffffffffffffffull

// CTA-collective insert of v (when valid) into the global hash set; distinct values are compacted into uniq[] with ONE atomicAdd per CTA
// (one per warp put ~900 same-address atomics on the critical path of the grid barrier that follows).  s_scratch: >= 34 ints of shared memory.
__device__ __forceinline__ void l1_set_insert(unsigned long long* __restrict__ table, unsigned table_mask, double* __restrict__ uniq, int* __restrict__ n_unique, double v, bool valid,
                                              int* s_scratch) {
  bool is_new = false;
  if (valid && v < INFINITY) {   // +inf = invalid slot, NaN never compares
    const unsigned long long key = (unsigned long long)__double_as_longlong(v == 0.0 ? 0.0 : v);   // -0.0 == 0.0 in a std::set
    unsigned h = (unsigned)((key * 0x9E3779B97F4A7C15ull) >> 40) & table_mask;
    for (;;) {
      const unsigned long long prev = atomicCAS(&table[h], L1_EMPTY, key);
      if (prev == L1_EMPTY) { is_new = true; break; }
      if (prev == key) break;
      h = (h + 1) & table_mask;
    }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = (blockDim.x + 31) >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, is_new);
  if (lane == 0) s_scratch[warp] = __popc(m);
  __syncthreads();
  if (threadIdx.x == 0) { int tot = 0; for (int w = 0; w < nwarp; w++) { const int c = s_scratch[w]; s_scratch[w] = tot; tot += c; } s_scratch[32] = tot ? atomicAdd(n_unique, tot) : 0; }
  __syncthreads();
  if (is_new) uniq[s_scratch[32] + s_scratch[warp] + __popc(m & ((1u << lane) - 1u))] = v == 0.0 ? 0.0 : v;   // +0.0 for a -0.0: block_select ranks bit patterns
  __syncthreads();
}

// Bit pattern of a non-negative double as an order-preserving key (-0.0 == 0.0 in a std::set).
__device__ __forceinline__ unsigned long long l1_key(double v) { return (unsigned long long)__double_as_longlong(v == 0.0 ? 0.0 : v); }
// Insert without compaction: true when this call created the entry, i.e. the caller is the (only) representative of a distinct value.
__device__ __forceinline__ bool l1_set_insert_flag(unsigned long long* __restrict__ table, unsigned table_mask, double v, bool valid) {
  if (!(valid && v < INFINITY)) return false;   // +inf = invalid slot, NaN never compares
  const unsigned long long key = l1_key(v);
  unsigned h = (unsigned)((key * 0x9E3779B97F4A7C15ull) >> 40) & table_mask;
  for (;;) {
    const unsigned long long prev = atomicCAS(&table[h], L1_EMPTY, key);
    if (prev == L1_EMPTY) return true;
    if (prev == key) return false;
    h = (h + 1) & table_mask;
  }
}

// Block-collective (NT threads): the k-th smallest (k = min(floor(ratio n), n-1)) of uniq[0..n) — distinct non-negative doubles, whose bit patterns
// order like the values.  11-bit digits from the top; as soon as the bin holding the k-th element has <= 1024 members they are gathered and ranked
// directly, which for a scan's L1 norms happens after two passes.  Returns the value to every thread.  n >= 1.
struct SelectSmem { unsigned hist[2048]; unsigned long long list[1024]; unsigned warp_sum[36]; unsigned long long red_and[32], red_or[32]; unsigned long long prefix, mask, result; int k, m, cnt, top; };
template <int NT>
__device__ double block_select(const double* __restrict__ uniq, int n, double ratio, SelectSmem& S) {
  constexpr int BPT = 2048 / NT;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // Pre-pass: the bits all keys share.  The norms of one scan span a few binades, so the top ~10 bits are common; starting the digits below
  // them spreads the keys over the 2048 bins (digits on the common exponent put 28k shared-memory atomics on 3 addresses).
  unsigned long long kand = ~0ull, kor = 0ull;
  for (int base0 = 0; base0 < n; base0 += NT * 8) {
    unsigned long long key[8];
#pragma unroll
    for (int u = 0; u < 8; u++) { const int i = base0 + u * NT + tid; key[u] = i < n ? (unsigned long long)__double_as_longlong(__ldcg(uniq + i)) : 0ull; }
#pragma unroll
    for (int u = 0; u < 8; u++) if (base0 + u * NT + tid < n) { kand &= key[u]; kor |= key[u]; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { kand &= __shfl_xor_sync(0xffffffffu, kand, o); kor |= __shfl_xor_sync(0xffffffffu, kor, o); }
  if (lane == 0) { S.red_and[warp] = kand; S.red_or[warp] = kor; }
  __syncthreads();
  if (tid == 0) {
    unsigned long long a = ~0ull, o = 0ull;
    for (int w = 0; w < NT / 32; w++) { a &= S.red_and[w]; o |= S.red_or[w]; }
    const unsigned long long diff = a ^ o;
    const int top = diff ? 63 - __clzll((long long)diff) : -1;            // highest bit on which two keys differ
    const unsigned long long hi = top >= 63 ? 0ull : (top < 0 ? ~0ull : (~0ull << (top + 1)));
    int k = (int)(ratio * (double)n); if (k > n - 1) k = n - 1;
    S.k = k; S.prefix = a & hi; S.mask = hi; S.m = n; S.cnt = 0; S.result = 0ull; S.top = top;
  }
  __syncthreads();
  while (S.m > 1024 && S.top >= 0) {
    const int top = S.top, shift = top >= 10 ? top - 10 : 0; const unsigned dmask = (1u << (top - shift + 1)) - 1u;
#pragma unroll
    for (int b = 0; b < BPT; b++) S.hist[tid * BPT + b] = 0u;
    __syncthreads();
    const unsigned long long prefix = S.prefix, himask = S.mask;
    for (int base0 = 0; base0 < n; base0 += NT * 8) {   // 8 independent loads in flight per thread (latency-bound pass)
      unsigned long long key[8];
#pragma unroll
      for (int u = 0; u < 8; u++) { const int i = base0 + u * NT + tid; key[u] = i < n ? (unsigned long long)__double_as_longlong(__ldcg(uniq + i)) : ~0ull; }
#pragma unroll
      for (int u = 0; u < 8; u++) if (base0 + u * NT + tid < n && (key[u] & himask) == prefix) atomicAdd(&S.hist[(unsigned)(key[u] >> shift) & dmask], 1u);
    }
    __syncthreads();
    unsigned h[BPT], run = 0;
#pragma unroll
    for (int b = 0; b < BPT; b++) { h[b] = S.hist[tid * BPT + b]; run += h[b]; }
    unsigned incl = run;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
    if (lane == 31) S.warp_sum[warp] = incl;
    __syncthreads();
    if (warp == 0) { unsigned w = lane < NT / 32 ? S.warp_sum[lane] : 0u, wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const unsigned v = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += v; }
      S.warp_sum[lane] = wi - w; }
    __syncthreads();
    const unsigned excl = S.warp_sum[warp] + incl - run; const unsigned k = (unsigned)S.k;
    __syncthreads();
    if (k >= excl && k < excl + run) {   // exactly one thread
      unsigned below = excl; int j = 0;
#pragma unroll
      for (int b = 0; b < BPT; b++) { if (k >= below + h[b] && j == b) { below += h[b]; j = b + 1; } }
      S.k = (int)(k - below); S.m = (int)h[j < BPT ? j : BPT - 1];
      S.prefix = prefix | ((unsigned long long)(tid * BPT + j) << shift);
      S.mask = himask | ((unsigned long long)dmask << shift);
      S.top = shift - 1;
    }
    __syncthreads();
  }
  const unsigned long long prefix = S.prefix, himask = S.mask;
  for (int base0 = 0; base0 < n; base0 += NT * 8) {
    unsigned long long key[8];
#pragma unroll
    for (int u = 0; u < 8; u++) { const int i = base0 + u * NT + tid; key[u] = i < n ? (unsigned long long)__double_as_longlong(__ldcg(uniq + i)) : ~0ull; }
#pragma unroll
    for (int u = 0; u < 8; u++) {
      const bool ok = base0 + u * NT + tid < n && (key[u] & himask) == prefix;
      const unsigned act = __ballot_sync(0xffffffffu, ok);
      if (act) {
        const int leader = __ffs(act) - 1; int slot0 = 0;
        if (lane == leader) slot0 = atomicAdd(&S.cnt, __popc(act));
        slot0 = __shfl_sync(0xffffffffu, slot0, leader);
        const int slot = slot0 + __popc(act & ((1u << lane) - 1u));
        if (ok && slot < 1024) S.list[slot] = key[u];
      }
    }
  }
  __syncthreads();
  const int m = min(S.cnt, 1024);
  for (int e = tid; e < m; e += NT) {
    const unsigned long long mine = S.list[e]; int rank = 0;
    for (int q = 0; q < m; q++) rank += (S.list[q] < mine) ? 1 : 0;
    if (rank == S.k) S.result = mine;
  }
  __syncthreads();
  return __longlong_as_double((long long)S.result);
}
