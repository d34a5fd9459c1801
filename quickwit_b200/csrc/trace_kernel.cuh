// trace_kernel.cuh — the find_trace_ids collector (Jaeger trace search) on the device.
//
// Reference: quickwit-search/src/find_trace_ids_collector.rs. Per split (= per segment), for the matched docs in
// ascending doc id, SelectTraceIds keeps the latest span timestamp per trace-id ordinal in a map of at most 2N
// entries; a full map is cut to its top N by (timestamp desc, ordinal asc), and the N-th timestamp becomes a
// sentinel below which (inclusive) later spans are dropped. Its result equals E = the exact top N of the per-trace
// maxima except in two cases (DESIGN §4.7): the N-th and (N+1)-th maxima of E tie, or a span carries i64::MIN
// and is not the split's first matched doc (the initial sentinel is i64::MIN, so such a span is always dropped).
//
//   collect  (hook in k_window's generic collect, trace_collect below): every matched doc reads its ordinal (first
//            term ordinal of the bytes column, 0 when the doc has none) and timestamp (first value of the date
//            column, 0 ns when missing); adjacent lanes with equal ordinals are combined with a warp segmented max,
//            then one 64-bit atomicMax on the order-preserving timestamp into best[ordinal]. A span at i64::MIN
//            maps to 0 = "no span" and records (doc, ordinal) instead, for the first-doc rule; the window's match
//            bitmap is kept for the replay.
//   select   (k_trace_select, one block per split): radix select of the (N+1)-th largest timestamp over best[];
//            when fewer than N traces lie strictly above it the N-th and (N+1)-th tie and the split is flagged for
//            the replay, otherwise the traces above it are the result.
//   replay   (k_trace_replay, one block per flagged split; the others leave at once): the block compacts the
//            matched docs of 1024-doc tiles into shared memory in doc order, then one thread runs SelectTraceIds
//            over them doc by doc, with the <= 2N-entry map in shared memory and an ordinal -> slot index in the
//            (no longer needed) best[] array. Exact by construction.
//
// Results go to the split's QwAggCell[N] (QW_AGG_TRACE_IDS in qwgpu_format.h); the host maps ordinals to trace
// ids and sorts.
#pragma once
#include "kernels.cuh"

namespace qwk {

struct DTraceState {  // per split, call scratch (initialised to 0xFF bytes)
  uint32_t first_doc;  // smallest matched doc id
  uint32_t pad;
  uint64_t min_span;   // smallest (doc << 32 | ordinal) among matched docs whose timestamp is i64::MIN
};

// ordinal + order-preserving timestamp of a matched doc (i64 0 maps to 1 << 63, i64::MIN to 0)
__device__ __forceinline__ void trace_doc(const DSplitPlan& P, const DCol* cols, const uint8_t* base, uint32_t doc, uint32_t& ord, uint64_t& ts) {
  uint64_t a, b;
  const DCol& oc = cols[P.tr_ord_col];
  col_range(base, oc, doc, a, b);
  ord = a < b ? (uint32_t)(oc.min_value + oc.gcd * col_raw(base, oc, a)) : 0u;
  ts = 1ull << 63;
  if (P.tr_ts_col != 0xFFFFFFFFu) {
    const DCol& tc = cols[P.tr_ts_col];
    col_range(base, tc, doc, a, b);
    if (a < b) ts = tc.min_value + tc.gcd * col_raw(base, tc, a);
  }
}

// warp-converged: lane = one doc (`on` = matched)
__device__ __forceinline__ void trace_collect(const DSplitPlan& P, const DCol* cols, const uint8_t* base, uint32_t doc, bool on, uint32_t lane) {
  uint32_t ord = 0xFFFFFFFFu;
  uint64_t ts = 0;
  if (on) trace_doc(P, cols, base, doc, ord, ts);
  DTraceState* st = (DTraceState*)P.tr_state;
  const uint32_t first = __reduce_min_sync(QW_FULL, on ? doc : 0xFFFFFFFFu);
  if (lane == 0 && first != 0xFFFFFFFFu) atomicMin(&st->first_doc, first);
  if (on && ts == 0) atomicMin((unsigned long long*)&st->min_span, ((unsigned long long)doc << 32) | ord);
  // segmented max: m covers the lanes [lane, end of lane's run of equal ordinals]
  uint64_t m = ts;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint64_t mo = __shfl_down_sync(QW_FULL, m, o);
    const uint32_t oo = __shfl_down_sync(QW_FULL, ord, o);
    if (lane + o < 32 && oo == ord && mo > m) m = mo;
  }
  const uint32_t prev = __shfl_up_sync(QW_FULL, ord, 1);
  if (on && (lane == 0 || prev != ord) && m != 0) atomicMax((unsigned long long*)P.tr_best + ord, (unsigned long long)m);
}

__device__ __forceinline__ void trace_emit(const DSplitPlan& P, uint32_t slot, uint32_t ord, uint64_t ts) {
  QwAggCell* c = (QwAggCell*)P.out_cells + slot;
  c->count = 1;
  c->sum_bits = ord;
  c->max_mapped = ts;
}

// the one ordinal whose only span is the split's first matched doc at i64::MIN (0xFFFFFFFF: none)
__device__ __forceinline__ uint32_t trace_min_ord(const DSplitPlan& P) {
  const DTraceState* st = (const DTraceState*)P.tr_state;
  const uint64_t ms = st->min_span;
  if (st->first_doc == 0xFFFFFFFFu || (uint32_t)(ms >> 32) != st->first_doc) return 0xFFFFFFFFu;
  const uint32_t o = (uint32_t)ms;
  return ((const uint64_t*)P.tr_best)[o] == 0 ? o : 0xFFFFFFFFu;
}

__global__ void __launch_bounds__(1024) k_trace_select(const DSplitPlan* plans) {
  const DSplitPlan& P = plans[blockIdx.x];
  if (!P.tr_on || P.tr_n == 0) return;
  __shared__ uint32_t s_hist[256];
  __shared__ uint64_t s_prefix;
  __shared__ uint32_t s_want, s_min_ord, s_out;
  const uint32_t tid = threadIdx.x, n = P.tr_num_ords;
  const uint64_t* best = (const uint64_t*)P.tr_best;
  if (tid == 0) { s_min_ord = trace_min_ord(P); s_out = 0; }
  __syncthreads();
  const uint32_t min_ord = s_min_ord;
  // present entries: best != 0, plus the first-doc i64::MIN span (key 0)
  uint32_t mine = 0;
  for (uint32_t i = tid; i < n; i += blockDim.x) mine += best[i] != 0;
  mine = __reduce_add_sync(QW_FULL, mine);
  if ((tid & 31) == 0 && mine) atomicAdd(&s_out, mine);
  __syncthreads();
  const uint32_t total = s_out + (min_ord != 0xFFFFFFFFu ? 1u : 0u);
  __syncthreads();
  if (tid == 0) s_out = 0;
  const uint32_t N = P.tr_n;
  if (total <= N) {
    // every trace is in the result
    __syncthreads();
    for (uint32_t i = tid; i < n; i += blockDim.x)
      if (best[i] != 0) trace_emit(P, atomicAdd(&s_out, 1u), i, best[i]);
    if (tid == 0 && min_ord != 0xFFFFFFFFu) trace_emit(P, atomicAdd(&s_out, 1u), min_ord, 0);
    return;
  }
  // radix select, 8 bits per pass: T = the (N+1)-th largest key among the present entries
  uint64_t prefix = 0;
  uint32_t want = N + 1, above = 0;
  for (int sh = 56; sh >= 0; sh -= 8) {
    for (uint32_t i = tid; i < 256; i += blockDim.x) s_hist[i] = 0;
    __syncthreads();
    const uint64_t hi_mask = sh == 56 ? 0ull : (~0ull << (sh + 8));
    for (uint32_t i = tid; i < n; i += blockDim.x) {
      const uint64_t k = best[i];
      if (k != 0 && (k & hi_mask) == prefix) atomicAdd(&s_hist[(uint32_t)(k >> sh) & 255u], 1u);
    }
    if (tid == 0 && min_ord != 0xFFFFFFFFu && (0ull & hi_mask) == prefix) atomicAdd(&s_hist[0], 1u);
    __syncthreads();
    if (tid == 0) {
      uint32_t acc = 0, d = 255;
      for (;; d--) {
        if (acc + s_hist[d] >= want) break;
        acc += s_hist[d];
      }
      s_prefix = prefix | ((uint64_t)d << sh);
      s_want = want - acc;
      s_hist[0] = acc;  // (read back below; every thread has left the counting loop)
    }
    __syncthreads();
    above += s_hist[0];
    prefix = s_prefix;
    want = s_want;
    __syncthreads();
  }
  const uint64_t T = prefix;
  // above = entries with key > T; a tie between the N-th and (N+1)-th iff above < N
  if (above < N) {
    if (tid == 0) *(uint32_t*)P.tr_tie = 1;
    return;
  }
  for (uint32_t i = tid; i < n; i += blockDim.x)
    if (best[i] > T) trace_emit(P, atomicAdd(&s_out, 1u), i, best[i]);
}

// ---- replay -----------------------------------------------------------------------------------------------
struct TraceMap {
  uint32_t* ord;  // shared memory, 2N entries
  uint64_t* ts;
  uint32_t* slot;  // global: ordinal -> map index + 1 (0 = absent)
  uint32_t m, N;
  uint64_t sentinel;

  __device__ __forceinline__ bool better(uint32_t a, uint32_t b) const {
    return ts[a] > ts[b] || (ts[a] == ts[b] && ord[a] < ord[b]);
  }
  __device__ __forceinline__ void swap(uint32_t a, uint32_t b) {
    const uint32_t o = ord[a]; ord[a] = ord[b]; ord[b] = o;
    const uint64_t t = ts[a]; ts[a] = ts[b]; ts[b] = t;
  }
  __device__ void dedup(uint32_t o, uint64_t t) {
    const uint32_t s = slot[o];
    if (s) { if (ts[s - 1] < t) ts[s - 1] = t; return; }
    ord[m] = o; ts[m] = t; slot[o] = ++m;
  }
  // select_nth_unstable(k - 1) by (ts desc, ord asc): the best k entries end up in [0, k)
  __device__ void select(uint32_t k) {
    uint32_t lo = 0, hi = m - 1;
    while (lo < hi) {
      const uint32_t mid = lo + (hi - lo) / 2;
      // median of three as pivot, moved to hi
      if (better(mid, lo)) swap(mid, lo);
      if (better(hi, lo)) swap(hi, lo);
      if (better(mid, hi)) swap(mid, hi);
      uint32_t store = lo;
      for (uint32_t i = lo; i < hi; i++)
        if (better(i, hi)) swap(i, store++);
      swap(store, hi);
      if (store == k - 1) break;
      if (store < k - 1) lo = store + 1; else hi = store - 1;
    }
  }
  __device__ void truncate() {
    if (m < 2 * N) return;
    select(N);
    sentinel = ts[N - 1];
    for (uint32_t i = N; i < m; i++) slot[ord[i]] = 0;
    for (uint32_t i = 0; i < N; i++) slot[ord[i]] = i + 1;
    m = N;
  }
};

#define QT_TILE 1024
__global__ void __launch_bounds__(QT_TILE) k_trace_replay(const DSplitPlan* plans, const DCol* all_cols) {
  const DSplitPlan& P = plans[blockIdx.x];
  if (!P.tr_on || P.tr_n == 0 || *(const volatile uint32_t*)P.tr_tie == 0) return;
  extern __shared__ __align__(16) uint8_t smem[];
  const uint32_t N = P.tr_n, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint64_t* m_ts = (uint64_t*)smem;
  uint64_t* t_ts = m_ts + 2 * N;
  uint32_t* m_ord = (uint32_t*)(t_ts + QT_TILE);
  uint32_t* t_ord = m_ord + 2 * N;
  __shared__ uint32_t s_wcnt[QT_TILE / 32];
  __shared__ uint32_t s_cnt;
  const DCol* cols = all_cols + P.col_base;
  const uint8_t* base = (const uint8_t*)P.data_base;
  uint32_t* slot = (uint32_t*)P.tr_best;  // best[] is dead after k_trace_select: reused as the slot index
  for (uint32_t i = tid; i < P.tr_num_ords; i += QT_TILE) slot[i] = 0;
  __syncthreads();
  TraceMap map{m_ord, m_ts, slot, 0u, N, 0ull};
  bool running = false;
  uint32_t r_ord = 0;
  uint64_t r_ts = 0;
  const uint32_t* match = (const uint32_t*)P.match_out;
  for (uint32_t d0 = 0; d0 < P.num_docs; d0 += QT_TILE) {
    const uint32_t doc = d0 + tid;
    const bool on = doc < P.num_docs && ((match[doc >> 5] >> (doc & 31)) & 1u);
    uint32_t ord = 0;
    uint64_t ts = 0;
    if (on) trace_doc(P, cols, base, doc, ord, ts);
    const uint32_t bal = __ballot_sync(QW_FULL, on);
    if (lane == 0) s_wcnt[warp] = __popc(bal);
    __syncthreads();
    if (tid == 0) {
      uint32_t acc = 0;
      for (uint32_t w = 0; w < QT_TILE / 32; w++) { const uint32_t c = s_wcnt[w]; s_wcnt[w] = acc; acc += c; }
      s_cnt = acc;
    }
    __syncthreads();
    if (on) {
      const uint32_t p = s_wcnt[warp] + __popc(bal & ((1u << lane) - 1u));
      t_ord[p] = ord;
      t_ts[p] = ts;
    }
    __syncthreads();
    if (tid == 0) {
      // SelectTraceIds::collect, doc by doc (timestamps compared in the order-preserving mapping)
      const uint32_t cnt = s_cnt;
      for (uint32_t i = 0; i < cnt; i++) {
        const uint32_t o = t_ord[i];
        const uint64_t t = t_ts[i];
        if (!running) { running = true; r_ord = o; r_ts = t; continue; }
        if (map.sentinel >= t) continue;
        if (r_ord == o) { if (t > r_ts) r_ts = t; continue; }
        map.dedup(r_ord, r_ts);
        map.truncate();
        r_ord = o;
        r_ts = t;
      }
    }
    __syncthreads();
  }
  if (tid == 0) {
    // harvest: dedup the running trace, then the top min(N, m)
    if (running) map.dedup(r_ord, r_ts);
    if (map.m) {
      const uint32_t k = map.m < N ? map.m : N;
      map.select(k);
      for (uint32_t i = 0; i < k; i++) trace_emit(P, i, map.ord[i], map.ts[i]);
    }
  }
}

}  // namespace qwk
