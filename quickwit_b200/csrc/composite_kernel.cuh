// composite_kernel.cuh — k_composite_cut: the per-split cut of composite aggregations to `size` (DESIGN.md §4.4).
//
// Runs once per hashed collect pass, one block per split, after k_window has filled the split's hashed table and
// before the used entries are copied back. For each composite of the split's plan (a chain of source nodes flagged
// QW_AGG_COMP_LEVEL, the last one QW_AGG_COMP_LAST) it keeps the `size` leaf entries whose key tuples come first in
// the composite's order, the chain entries above them and every sub-aggregation entry below them. Entries of other
// aggregations stay. The kept entries are compacted in their original order, their parent indices rewritten, and the
// kept count replaces the split's counter, so the copy-back moves only them.
//
// The selection is an exact radix select over the tuple, most significant first: per source level a 1-bit digit (the
// null's place: first ascending, last descending), then eight 8-bit digits of the key (complemented when descending).
// Each pass histograms the digit over the leaves still tied with the prefix, fixes the digit where the rank `size`
// falls, keeps the leaves below it and drops those above. Tuples are unique (one leaf per path), so the pass that
// leaves exactly the remaining rank tied ends the selection.
//
// Scratch: the split's slot table (at least 2 * h_cap words) is dead once the collect pass has ended; its first
// h_cap words hold the per-entry selection state, then the new index of every entry; the next h_cap words the keep
// flags.
#pragma once
#include "device_types.h"

namespace qwk {

#define QC_THREADS 1024
enum { QC_NONE = 0, QC_ALIVE = 1, QC_KEEP = 2, QC_DROP = 3 };

// digit `b` (0: the null's place, 1..8: key bytes from the top) of an entry of composite level flags `comp`
__device__ __forceinline__ uint32_t qc_digit(uint32_t comp, const DHKey& k, uint32_t b) {
  const bool miss = (k.node_flags >> 8) & QW_AGG_ENTRY_MISSING;
  const bool desc = comp & QW_AGG_COMP_DESC;
  if (b == 0) return desc ? (miss ? 1u : 0u) : (miss ? 0u : 1u);
  const uint64_t v = miss ? 0ull : (desc ? ~k.key : k.key);
  return (uint32_t)(v >> (8 * (8 - b))) & 0xFFu;
}

// exclusive block-wide prefix sum of `x` (every thread calls it); returns the block total in `total`
__device__ __forceinline__ uint32_t qc_scan(uint32_t x, uint32_t* s_warp, uint32_t& total) {
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t v = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, v, o);
    if (lane >= (uint32_t)o) v += y;
  }
  if (lane == 31) s_warp[warp] = v;
  __syncthreads();
  if (warp == 0) {
    uint32_t w = lane < (QC_THREADS / 32) ? s_warp[lane] : 0u;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, w, o);
      if (lane >= (uint32_t)o) w += y;
    }
    s_warp[lane] = w;  // inclusive over warps
  }
  __syncthreads();
  total = s_warp[QC_THREADS / 32 - 1];
  const uint32_t before = (warp ? s_warp[warp - 1] : 0u) + v - x;
  __syncthreads();  // (s_warp is reused by the next call)
  return before;
}

__global__ void __launch_bounds__(QC_THREADS) k_composite_cut(const DSplitPlan* plans, const DAgg* all_aggs) {
  const DSplitPlan& P = plans[blockIdx.x];
  if (!P.hashed) return;
  const uint32_t ctr = *(volatile const uint32_t*)P.h_ctr;
  if (ctr >> 31) return;  // overflowed: the batch runs again at the bound
  const uint32_t used = min(ctr & 0x7FFFFFFFu, P.h_cap);
  const DAgg* aggs = all_aggs + P.agg_base;
  const uint32_t tid = threadIdx.x;
  __shared__ uint32_t s_comp[QW_MAX_AGG_NODES], s_chain[QW_MAX_AGG_LEVELS];
  __shared__ uint32_t s_hist[256], s_warp[32];
  __shared__ uint32_t s_k, s_sel, s_tied, s_n_leaves, s_any;
  if (tid < QW_MAX_AGG_NODES) s_comp[tid] = tid < P.n_aggs ? aggs[tid].comp : 0u;
  if (tid == 0) s_any = 0;
  __syncthreads();
  DHKey* keys = (DHKey*)P.h_keys;
  QwAggCell* cells = (QwAggCell*)P.h_cells;
  uint32_t* st = (uint32_t*)P.h_table;           // selection state, later the new index
  uint32_t* keep = (uint32_t*)P.h_table + P.h_cap;
  for (uint32_t e = tid; e < used; e += QC_THREADS) st[e] = QC_NONE;
  __syncthreads();

  for (uint32_t top = 0; top < P.n_aggs; top++) {
    if (aggs[top].parent != 0xFFFFFFFFu || !(s_comp[top] & QW_AGG_COMP_LEVEL)) continue;
    // the source chain; a malformed one, or a page whose `after` the walk could not apply, is not cut
    uint32_t n = 0, g = top;
    bool ok = true;
    while (true) {
      if (n >= QW_MAX_AGG_LEVELS || g >= P.n_aggs || !(s_comp[g] & QW_AGG_COMP_LEVEL) || (s_comp[g] & QW_AGG_COMP_AFTER_HOST)) { ok = false; break; }
      if (tid == 0) s_chain[n] = g;
      n++;
      if (s_comp[g] & QW_AGG_COMP_LAST) break;
      if (aggs[g].num_children != 1) { ok = false; break; }
      g = aggs[g].first_child;
    }
    __syncthreads();
    if (!ok) continue;
    const uint32_t last = s_chain[n - 1];
    const uint64_t size64 = aggs[top].range_to[0];
    const uint32_t size = size64 > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)size64;
    if (tid == 0) { s_n_leaves = 0; s_any = 1; }
    __syncthreads();
    uint32_t mine = 0;
    for (uint32_t e = tid; e < used; e += QC_THREADS)
      if ((keys[e].node_flags & 0xFFu) == last && cells[e].count) { st[e] = QC_ALIVE; mine++; }
    atomicAdd(&s_n_leaves, mine);
    __syncthreads();
    const uint32_t n_leaves = s_n_leaves;
    if (n_leaves <= size) {
      for (uint32_t e = tid; e < used; e += QC_THREADS) if (st[e] == QC_ALIVE) st[e] = QC_KEEP;
      __syncthreads();
      continue;
    }
    if (tid == 0) { s_k = size; s_tied = n_leaves; }
    __syncthreads();
    for (uint32_t d = 0; d < n && s_tied > s_k; d++) {
      const uint32_t comp = s_comp[s_chain[d]];
      for (uint32_t b = 0; b < 9 && s_tied > s_k; b++) {
        for (uint32_t v = tid; v < 256; v += QC_THREADS) s_hist[v] = 0;
        __syncthreads();
        for (uint32_t e = tid; e < used; e += QC_THREADS) {
          if (st[e] != QC_ALIVE) continue;
          uint32_t x = e;
          for (uint32_t j = n - 1; j > d; j--) x = keys[x].parent;
          atomicAdd(&s_hist[qc_digit(comp, keys[x], b)], 1u);
        }
        __syncthreads();
        if (tid == 0) {
          uint32_t cum = 0, v = 0;
          for (; v < 255 && cum + s_hist[v] < s_k; v++) cum += s_hist[v];
          s_sel = v;
          s_k -= cum;
          s_tied = s_hist[v];
        }
        __syncthreads();
        const uint32_t sel = s_sel;
        for (uint32_t e = tid; e < used; e += QC_THREADS) {
          if (st[e] != QC_ALIVE) continue;
          uint32_t x = e;
          for (uint32_t j = n - 1; j > d; j--) x = keys[x].parent;
          const uint32_t dg = qc_digit(comp, keys[x], b);
          if (dg < sel) st[e] = QC_KEEP;
          else if (dg > sel) st[e] = QC_DROP;
        }
        __syncthreads();
      }
    }
    // the leaves still tied hold exactly the remaining rank
    for (uint32_t e = tid; e < used; e += QC_THREADS) if (st[e] == QC_ALIVE) st[e] = QC_KEEP;
    __syncthreads();
  }
  if (!s_any) return;

  // keep flags: an entry at or below a composite leaf follows that leaf; composite chain entries above the leaves
  // are kept by the kept leaves below them; every other entry stays
  for (uint32_t e = tid; e < used; e += QC_THREADS) {
    uint32_t k = 1, x = e;
    for (uint32_t hop = 0; hop <= QW_MAX_AGG_LEVELS && x != QW_AGG_NO_PARENT; hop++) {
      const uint32_t c = s_comp[keys[x].node_flags & 0xFFu];
      if (c & QW_AGG_COMP_LAST) { k = st[x] == QC_DROP ? 0u : 1u; break; }
      if ((c & QW_AGG_COMP_LEVEL) && x == e) k = 0;  // above the leaves: decided by them
      x = keys[x].parent;
    }
    keep[e] = k;
  }
  __syncthreads();
  for (uint32_t e = tid; e < used; e += QC_THREADS) {
    if (!(s_comp[keys[e].node_flags & 0xFFu] & QW_AGG_COMP_LAST) || st[e] == QC_DROP) continue;
    for (uint32_t x = keys[e].parent; x != QW_AGG_NO_PARENT; x = keys[x].parent) keep[x] = 1;
  }
  __syncthreads();
  // new indices (exclusive prefix sum of the keep flags, in entry order)
  uint32_t carry = 0;
  for (uint32_t base = 0; base < used; base += QC_THREADS) {
    const uint32_t e = base + tid;
    const uint32_t f = e < used ? keep[e] : 0u;
    uint32_t total;
    const uint32_t before = qc_scan(f, s_warp, total);
    if (e < used) st[e] = carry + before;
    carry += total;
  }
  __syncthreads();
  // compact in place, a block-sized chunk at a time: every entry moves to a lower or equal index, and a chunk is read
  // whole before it is written
  for (uint32_t base = 0; base < used; base += QC_THREADS) {
    const uint32_t e = base + tid;
    const bool k = e < used && keep[e];
    DHKey key;
    QwAggCell cell;
    uint32_t to = 0;
    if (k) {
      key = keys[e];
      cell = cells[e];
      to = st[e];
      if (key.parent != QW_AGG_NO_PARENT) key.parent = st[key.parent];
    }
    __syncthreads();
    if (k) { keys[to] = key; cells[to] = cell; }
    __syncthreads();
  }
  if (tid == 0) *(volatile uint32_t*)P.h_ctr = carry;
}

}  // namespace qwk
