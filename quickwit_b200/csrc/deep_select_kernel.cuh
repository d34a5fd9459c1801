// deep_select_kernel.cuh — the final top-K selection of splits that ask for more than QW_MAX_TOPK hits.
//
// k_select holds every candidate's first key word in shared memory, which caps it at QW_CAND_CAP candidates and
// K <= QW_MAX_TOPK. A split with a larger K (max_hits + start_offset up to QW_MAX_HITS) keeps qw_cand_cap(K) = 2K
// (rounded up to 1024) candidates in call scratch and is finished here, in the same total order (the 192-bit composite
// key, greater = better; keys are unique within a split because they end in the doc id):
//   cut   (k_deep_cut, one block per split): MSB-first 8-bit radix select of the K-th largest first key word over the
//         candidates in global memory, then compaction of every candidate whose first word reaches it into a survivor
//         array (three word arrays of qw_cand_cap(K) entries) with one shared atomic per warp;
//   sort  (k_deep_sort, one block per 2048-survivor tile): bitonic sort of the tile in shared memory (48 KB), best
//         first, written back in place;
//   rank  (k_deep_rank, one thread per survivor): the survivor's final rank is its index in its own tile plus, for
//         every other tile, the number of keys there that beat it (one binary search per tile); the ranks form a
//         permutation, and a survivor ranked below K is decoded straight into the split's hit list (write_hit).
// Every kernel leaves at once for a split with K <= QW_MAX_TOPK (k_select's), and for tiles and survivors past the
// split's survivor count: the host launches the grids from capacities, without reading the counts back.
#pragma once
#include "kernels.cuh"

namespace qwk {

#define QD_TILE 2048  /* survivors per sorted tile: 3 x 2048 x 8 B = 48 KB of shared memory */

struct DeepSurvivors {
  uint64_t *k0, *k1, *k2;  // word arrays of the split's survivors (qw_cand_cap(K) entries each)
  __device__ __forceinline__ DeepSurvivors(const DSplitPlan& P, size_t surv_off) {
    const uint32_t cap = qw_cand_cap(P.max_hits);
    k0 = (uint64_t*)((uint8_t*)P.out_cands + surv_off);
    k1 = k0 + cap;
    k2 = k1 + cap;
  }
};

// surv_off: byte distance from a split's candidate list to its survivor arrays; deep_m[split]: survivor count
__global__ void __launch_bounds__(1024) k_deep_cut(const DSplitPlan* plans, size_t surv_off, uint32_t* deep_m) {
  const DSplitPlan& P = plans[blockIdx.x];
  const uint32_t tid = threadIdx.x, K = P.max_hits;
  if (K <= QW_MAX_TOPK) return;
  const uint32_t cap = qw_cand_cap(K);
  uint32_t n = *(const uint32_t*)P.out_cand_count;
  if (n > cap) n = cap;  // overflow is detected by the host (cand_count > cap)
  const uint64_t* src = (const uint64_t*)P.out_cands;
  const DeepSurvivors sv(P, surv_off);
  __shared__ uint32_t s_hist[256];
  __shared__ uint32_t s_sel[4];  // [0] digit, [1] count above digit, [2] survivor counter, [3] count in the digit's bin
  if (tid == 0) s_sel[2] = 0;
  uint64_t thr = 0;  // keep candidates with w0 >= thr
  if (n > K) {
    uint64_t prefix = 0;
    uint32_t need = K;  // rank of the wanted element among those matching the prefix
    // the sort works in whole tiles: once the candidates above the current bin plus the bin itself fit the tiles that
    // K survivors take anyway, the remaining digits need not be resolved (the whole bin is kept)
    const uint32_t keep = (K + QD_TILE - 1) / QD_TILE * QD_TILE;
    for (int shift = 56; shift >= 0; shift -= 8) {
      if (tid < 256) s_hist[tid] = 0;
      __syncthreads();
      const uint64_t himask = shift == 56 ? 0ull : (~0ull << (shift + 8));
      for (uint32_t base = 0; base < n; base += 1024) {
        const uint32_t i = base + tid;
        const uint64_t v = i < n ? src[3ull * i] : 0ull;
        const bool in = i < n && (v & himask) == prefix;
        const uint32_t bin = (uint32_t)(v >> shift) & 255u;
        const uint32_t act = __ballot_sync(0xFFFFFFFFu, in);
        if (in) {
          const uint32_t peers = __match_any_sync(act, bin);
          if ((tid & 31) == (uint32_t)__ffs(peers) - 1u) atomicAdd(&s_hist[bin], (uint32_t)__popc(peers));
        }
      }
      __syncthreads();
      if (tid < 32) {
        // lane owns 8 bins, top bins first: lane 0 -> bins 255..248
        uint32_t loc[8], sum = 0;
#pragma unroll
        for (int j = 0; j < 8; j++) { loc[j] = s_hist[255 - (tid * 8 + j)]; sum += loc[j]; }
        uint32_t incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, o); if ((int)tid >= o) incl += t; }
        uint32_t run = incl - sum;
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const uint32_t before = run;
          run += loc[j];
          if (before < need && run >= need) { s_sel[0] = 255 - (tid * 8 + j); s_sel[1] = before; s_sel[3] = loc[j]; }
        }
      }
      __syncthreads();
      prefix |= (uint64_t)s_sel[0] << shift;
      need -= s_sel[1];
      const uint32_t in_bin = s_sel[3];
      __syncthreads();
      if ((K - need) + in_bin <= keep) break;  // (block-uniform: every operand comes from shared memory)
    }
    thr = prefix;  // K-th largest first word with its unresolved low digits cleared: everything >= thr is kept
  }
  __syncthreads();
  for (uint32_t base = 0; base < n; base += 1024) {
    const uint32_t i = base + tid;
    const uint64_t v = i < n ? src[3ull * i] : 0ull;
    const bool kept = i < n && v >= thr;
    const uint32_t km = __ballot_sync(0xFFFFFFFFu, kept);  // one atomic per warp
    uint32_t wpos = 0;
    if ((tid & 31) == 0 && km) wpos = atomicAdd(&s_sel[2], (uint32_t)__popc(km));
    wpos = __shfl_sync(0xFFFFFFFFu, wpos, 0);
    if (kept) {
      const uint32_t pos = wpos + __popc(km & ((1u << (tid & 31)) - 1u));
      sv.k0[pos] = v; sv.k1[pos] = src[3ull * i + 1]; sv.k2[pos] = src[3ull * i + 2];
    }
  }
  __syncthreads();
  if (tid == 0) {
    const uint32_t m = s_sel[2];
    deep_m[blockIdx.x] = m;
    *(uint32_t*)P.out_nhits = m < K ? m : K;
  }
}

// grid (tiles of the largest deep capacity, splits)
__global__ void __launch_bounds__(1024) k_deep_sort(const DSplitPlan* plans, size_t surv_off, const uint32_t* deep_m) {
  const DSplitPlan& P = plans[blockIdx.y];
  const uint32_t tid = threadIdx.x;
  if (P.max_hits <= QW_MAX_TOPK) return;
  const uint32_t m = deep_m[blockIdx.y], base = blockIdx.x * QD_TILE;
  if (base >= m) return;
  const uint32_t len = min(m - base, (uint32_t)QD_TILE);
  const DeepSurvivors sv(P, surv_off);
  uint64_t* k0 = (uint64_t*)qw_smem;
  uint64_t* k1 = k0 + QD_TILE;
  uint64_t* k2 = k1 + QD_TILE;
  for (uint32_t i = tid; i < QD_TILE; i += 1024) {
    // (padding keys are zero: they sort last, and only the tile's first len entries are written back)
    if (i < len) { k0[i] = sv.k0[base + i]; k1[i] = sv.k1[base + i]; k2[i] = sv.k2[base + i]; }
    else { k0[i] = 0; k1[i] = 0; k2[i] = 0; }
  }
  __syncthreads();
  // bitonic network, descending: one compare-exchange per thread and step
  for (uint32_t size = 2; size <= QD_TILE; size <<= 1) {
    for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
      const uint32_t pos = 2 * tid - (tid & (stride - 1)), q = pos + stride;
      const bool desc = (pos & size) == 0;
      const Key a{k0[pos], k1[pos], k2[pos]}, b{k0[q], k1[q], k2[q]};
      if (desc ? key_lt(a, b) : key_lt(b, a)) {
        k0[pos] = b.w0; k1[pos] = b.w1; k2[pos] = b.w2;
        k0[q] = a.w0; k1[q] = a.w1; k2[q] = a.w2;
      }
      __syncthreads();
    }
  }
  for (uint32_t i = tid; i < len; i += 1024) { sv.k0[base + i] = k0[i]; sv.k1[base + i] = k1[i]; sv.k2[base + i] = k2[i]; }
}

// grid (survivors of the largest deep capacity / 256, splits)
__global__ void __launch_bounds__(256) k_deep_rank(const DSplitPlan* plans, const DCol* all_cols, size_t surv_off, const uint32_t* deep_m) {
  const DSplitPlan& P = plans[blockIdx.y];
  const uint32_t K = P.max_hits;
  if (K <= QW_MAX_TOPK) return;
  const uint32_t m = deep_m[blockIdx.y], j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= m) return;
  const uint32_t t = j / QD_TILE, n_tiles = (m + QD_TILE - 1) / QD_TILE;
  uint32_t r = j % QD_TILE;  // keys of the own tile that beat this one
  if (r >= K) return;
  const DeepSurvivors sv(P, surv_off);
  const Key key{sv.k0[j], sv.k1[j], sv.k2[j]};
  auto beats = [&](uint32_t i) {  // survivor i's key > key (mostly decided by the first word)
    const uint64_t a0 = sv.k0[i];
    if (a0 != key.w0) return a0 > key.w0;
    const uint64_t a1 = sv.k1[i];
    if (a1 != key.w1) return a1 > key.w1;
    return sv.k2[i] > key.w2;
  };
  for (uint32_t t2 = 0; t2 < n_tiles && r < K; t2++) {
    if (t2 == t) continue;
    const uint32_t base = t2 * QD_TILE;
    uint32_t lo = 0, hi = min(m - base, (uint32_t)QD_TILE);  // first index whose key does not beat `key`
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      if (beats(base + mid)) lo = mid + 1; else hi = mid;
    }
    r += lo;
  }
  if (r < K) write_hit(P, all_cols + P.col_base, key, r);
}

}  // namespace qwk
