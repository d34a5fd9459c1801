// driver_kernel.cuh — posting-driven evaluation of "one term AND column filters" queries.
//
// The window engine (kernels.cuh) pays per doc-id window: bitmaps to clear, a program to interpret, a block-wide
// barrier per clause, a sweep over the window at collect time. A query whose matches all come from ONE posting
// list — a single term (BASELINE config 1), or a required term narrowed by fast-field range / exists filters
// (config 3: term AND timestamp range, top-K by timestamp) — touches a few percent of the docs, and the window
// overheads dominate. This kernel walks the term's posting blocks instead, one warp per 128-posting block:
//   decode doc ids (+ tfs)  ->  per posting: probe the filter columns  ->  count the hit
//   MODE_HIST:    11-bit digit of the composite sort key -> the split's radix histogram
//   MODE_COLLECT: cheap 11-bit pre-filter, then the full key against the threshold -> candidate list
// Work is proportional to the postings of the driving term; there is no per-window state at all.
// Replaces, for these shapes, the same tantivy loop as the window engine: TermScorer / Intersection with
// FastFieldRangeQuery docsets + QuickwitSegmentCollector::collect (quickwit-search/src/leaf.rs:637,
// collector.rs:373-470). Same composite key, same threshold / radix select / k_select as the other paths.
#pragma once
#include "kernels.cuh"

namespace qwk {

#define QD_WARPS 8
#define QD_MAX_FILTERS 4

struct DrvParams {
  const DSplitPlan* plans;
  const DInstr* instrs;
  const DCol* cols;
  const DThresh* thresh;
  DWorkList wl;                // (split, posting block of the driving term) list; sampled passes: the sampled blocks
  uint32_t level, use_prefix;  // MODE_HIST
};

template <int MODE>
__global__ void __launch_bounds__(QD_WARPS * 32) k_driver(const DrvParams p) {
  __shared__ uint32_t s_hist[QW_HIST_BINS];
  __shared__ unsigned long long s_cnt[2];  // hits, eligible of the current split
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // this block's chunk of the flat (split, posting block) list
  const uint32_t w_begin = qw_chunk_begin(p.wl.total_work, blockIdx.x, gridDim.x);
  const uint32_t w_end = qw_chunk_begin(p.wl.total_work, blockIdx.x + 1, gridDim.x);
  if (w_begin >= w_end) return;
  uint32_t split = work_split(p.wl, w_begin);
  if (MODE == MODE_HIST) for (uint32_t i = tid; i < QW_HIST_BINS; i += QD_WARPS * 32) s_hist[i] = 0;
  if (tid < 2) s_cnt[tid] = 0;
  __syncthreads();

  for (uint32_t seg = w_begin; seg < w_end;) {
    while (__ldg(p.wl.first_work + split + 1) <= seg) split++;
    const uint32_t fw = __ldg(p.wl.first_work + split);
    const uint32_t seg_end = min(w_end, __ldg(p.wl.first_work + split + 1));
    const DSplitPlan& P = p.plans[split];
    const DKeySpec& ks = P.key;
    const DCol* cols = p.cols + P.col_base;
    const uint8_t* base = (const uint8_t*)P.data_base;
    const DInstr* prog = p.instrs + P.instr_base;  // [BOOL_BEGIN, TERM, filter x n, BOOL_END]
    const DInstr& term = prog[1];
    const uint32_t n_filters = P.n_instr - 3;
    const DThresh& T = p.thresh[split];
    const Key thr{T.key[0], T.key[1], T.key[2]};
    const uint32_t thr_top = (uint32_t)(thr.w0 >> 53);
    const bool scored = (term.flags & IF_SCORED) != 0;
    const bool has_tf = (term.flags & IF_HAS_TF) != 0, has_fn = (term.flags & IF_HAS_FN) != 0;
    const float* tab = (const float*)P.bm25_tab[term.r];
    const QwSkip* skips = (const QwSkip*)(base + term.c);
    const uint8_t* tdata = base + term.a;
    const uint32_t sa_present = P.sa.present, max_hits = P.max_hits;
    uint32_t my_hits = 0, my_elig = 0;

    for (uint32_t w = seg + warp; w < seg_end; w += QD_WARPS) {
      const uint32_t bb = qw_sample_item(w - fw, split, p.wl.stride);
      const uint8_t* blk = tdata + __ldg(&skips[bb].byte_off);
      const BlkHdr h = blk_header<LdgLoad>(blk);
      uint32_t doc[4], tf[4] = {1, 1, 1, 1};
      blk_docs<LdgLoad>(blk, h, 0, lane, doc);
      if (scored && has_tf) blk_tfs<LdgLoad>(blk, h, lane, tf);
      uint32_t fnw = 0x01010101u;  // no fieldnorms: constant fieldnorm id 1
      if (scored && has_fn) fnw = __ldg(reinterpret_cast<const uint32_t*>(blk + 16u + 16u * (h.doc_bits + h.tf_bits)) + lane);

#pragma unroll
      for (int j = 0; j < 4; j++) {
        bool on = lane * 4 + j < h.count;
        // ---- required column filters (FastFieldRangeQuery / ExistsQuery docsets) ------------------------------
        for (uint32_t f = 0; f < n_filters && on; f++) {
          const DInstr& fi = prog[2 + f];
          if (fi.r == 0xFFFFFFFFu) { on = false; break; }  // column absent from the split: nothing matches
          on = col_match(base, cols[fi.r], doc[j], fi.op, fi.a, fi.op == OP_COL_SET ? fi.n : fi.b);
        }
        my_hits += on ? 1u : 0u;
        if (!max_hits) continue;
        // ---- BM25 of the posting: weight * tf-factor (Bm25Weight::score) --------------------------------------
        float sc = 0.0f;
        if (scored && on) sc = __fmul_rn(term.f, tf_factor(tab, tf[j], (fnw >> (8 * j)) & 0xFFu));
        if (MODE == MODE_COLLECT) {
          uint32_t top;
          if (on) my_elig += rank_collect(P, ks, cols, base, doc[j], sc, sa_present, thr, thr_top, top);
        } else rank_hist(s_hist, P, ks, cols, base, doc[j], sc, on, sa_present, p.level, p.use_prefix, T, lane);
      }
    }

    // ---- end of this split's segment: counters and histogram go out ---------------------------------------------
    if (MODE == MODE_COLLECT) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        my_hits += __shfl_down_sync(QW_FULL, my_hits, o);
        my_elig += __shfl_down_sync(QW_FULL, my_elig, o);
      }
      if (lane == 0) {
        if (my_hits) atomicAdd(&s_cnt[0], (unsigned long long)my_hits);
        if (my_elig) atomicAdd(&s_cnt[1], (unsigned long long)my_elig);
      }
    }
    __syncthreads();
    if (MODE == MODE_COLLECT) {
      if (tid == 0) {
        flush_counts(P, sa_present, max_hits, s_cnt[0], s_cnt[1]);
        s_cnt[0] = s_cnt[1] = 0;
      }
    } else flush_hist(P, s_hist, 1, true, tid, QD_WARPS * 32);
    __syncthreads();
    seg = seg_end;
  }
}

}  // namespace qwk
