// agg_kernel.cuh — streaming bucket aggregations over a dense match set (match_all + flat terms /
// histogram / date_histogram nodes, no hits requested): BASELINE config C4.
//
// Replaces tantivy's AggregationSegmentCollector::collect_block over every doc of the segment
// (quickwit-search/src/collector.rs:782-791, 539-541; semantics docs/reference/aggregation.md:150-185,
// 500-560; SURVEY.md §8a row a12) for the case where nothing has to be decoded but the fast-field
// columns themselves: the kernel is a pure stream over the bit-packed columns.
//
//   producer warp   per chunk of 8192 docs: one `cp.async.bulk` (1-D TMA) per aggregated column copies
//                   the chunk's packed bytes (8192 * bits / 8, contiguous, 16-byte aligned) into the next
//                   slot of a 4-deep shared-memory ring; completion on the slot's `full` mbarrier.
//   consumer warps  one thread = one GROUP of 32 consecutive docs = exactly `bits` 32-bit words of a
//                   column: the words are read once from shared memory (stride `bits` words between
//                   lanes) and unpacked in registers by code specialised for the width.
//     histogram     a bucket is located in RAW space through the host-built boundary table (DAgg::bounds,
//                   computed with the reference f64 formula, monotone in the raw value). The bucket is
//                   monotone too, so a group whose smallest and largest raw value fall into the same
//                   bucket lies in it entirely — whatever the order of the docs: unpack + min/max costs
//                   ~3 instructions per doc, the two table searches are per GROUP, and a warp whose 32
//                   groups agree adds 1024 to one counter. Groups that straddle a boundary (or the hard
//                   bounds) take the per-doc path. Bit-exact by construction: every doc is counted in
//                   the bucket the boundary table assigns to its raw value.
//     terms         1- and 2-bit columns (e.g. severity_text) are counted with bit-plane popcounts, 32
//                   docs in ~10 instructions; wider columns add one shared-memory atomic per doc.
//   counters        privatised per block in shared memory, flushed to the split's cells with 64-bit
//                   global atomics when the block leaves the split.
#pragma once
#include "kernels.cuh"
#include "union_kernel.cuh"

namespace qwk {

#define QA_CW 8                  /* consumer warps; warp QA_CW is the producer */
#define QA_THREADS ((QA_CW + 1) * 32)
#define QA_GROUPS (QA_CW * 32)   /* 32-doc groups per chunk: one per consumer thread */
#define QA_CHUNK (QA_GROUPS * 32)
#define QA_SLOTS 2               /* per block; four blocks per SM keep eight chunks in flight */
#define QA_MINB 4
#define QA_MAX_CELLS 4096
#define QA_MAX_AGGS 8            /* aggregation nodes per plan: one column staged per node, indexed by lane & 7 */

struct ASmem {
  uint32_t slot0, slot_stride;
  uint32_t col_off[QA_MAX_AGGS];   // bytes of aggregation i's column inside a slot
  uint32_t hdr;                    // uint4 {split, first doc, docs, flags} inside a slot
  uint32_t bars;                   // full[QA_SLOTS], empty[QA_SLOTS]
  uint32_t atab;                   // AggRow[QA_MAX_AGGS]: the current split's aggregations
  uint32_t bcache;                 // uint4[QA_CW][QA_MAX_AGGS]: per warp, the histogram bucket it is in
  uint32_t cells;                  // uint32[n_cells]
  uint32_t total;
};

struct AParams {
  const DSplitPlan* plans;
  const DCol* cols;
  const DAgg* aggs;
  DWorkList wl;  // (split, chunk of QA_CHUNK docs) list
  ASmem sm;
};

struct AggRow {  // 48 bytes
  uint32_t kind, bits, cell_base, nb;
  float inv_step;
  uint32_t pad;
  uint64_t bounds;  // device address of uint64[nb + 1]
  uint64_t b0, bn;  // bounds[0], bounds[nb]
};

// 32 values of a group, bit-packed little-endian at B bits (tantivy-bitpacker layout), words in registers
template <int B, class F>
__device__ __forceinline__ void unpack32(const uint32_t* w, F&& f) {
  uint32_t r[B + 1];
#pragma unroll
  for (int i = 0; i < B; i++) r[i] = w[i];
  r[B] = 0;
  constexpr uint32_t mask = B >= 32 ? 0xFFFFFFFFu : ((1u << (B & 31)) - 1u);
#pragma unroll
  for (int v = 0; v < 32; v++) {
    const int bitpos = v * B, wi = bitpos >> 5, sh = bitpos & 31;
    uint32_t x = r[wi] >> sh;
    if (sh + B > 32) x |= r[wi + 1] << (32 - sh);
    f(v, x & mask);
  }
}
template <class F>
__device__ __forceinline__ void unpack32_dyn(uint32_t bits, const uint32_t* w, F&& f) {
  switch (bits) {
#define QA_CASE(B) case B: unpack32<B>(w, f); break;
    QA_CASE(1) QA_CASE(2) QA_CASE(3) QA_CASE(4) QA_CASE(5) QA_CASE(6) QA_CASE(7) QA_CASE(8)
    QA_CASE(9) QA_CASE(10) QA_CASE(11) QA_CASE(12) QA_CASE(13) QA_CASE(14) QA_CASE(15) QA_CASE(16)
    QA_CASE(17) QA_CASE(18) QA_CASE(19) QA_CASE(20) QA_CASE(21) QA_CASE(22) QA_CASE(23) QA_CASE(24)
    QA_CASE(25) QA_CASE(26) QA_CASE(27) QA_CASE(28) QA_CASE(29) QA_CASE(30) QA_CASE(31) QA_CASE(32)
#undef QA_CASE
    default: break;
  }
}

__global__ void __launch_bounds__(QA_THREADS, QA_MINB) k_aggscan(const AParams p) {
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // col_off is indexed at run time, which puts the indexed struct in local memory: a copy of the layout keeps that to
  // the layout instead of all of p
  const ASmem sm = p.sm;
  const uint32_t sbase = smem_u32(qw_smem);
  const uint32_t bars = sbase + sm.bars;
  auto bar_full = [&](uint32_t s) { return bars + 8u * s; };
  auto bar_empty = [&](uint32_t s) { return bars + 8u * (QA_SLOTS + s); };
  uint32_t* cells = (uint32_t*)(qw_smem + sm.cells);
  AggRow* atab = (AggRow*)(qw_smem + sm.atab);
  if (tid == 0) {
    for (uint32_t s = 0; s < QA_SLOTS; s++) { mbar_init(bar_full(s), 1); mbar_init(bar_empty(s), QA_CW); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  const uint32_t w_begin = qw_chunk_begin(p.wl.total_work, blockIdx.x, gridDim.x);
  const uint32_t w_end = qw_chunk_begin(p.wl.total_work, blockIdx.x + 1, gridDim.x);
  uint32_t split = work_split(p.wl, w_begin);

  if (warp == QA_CW) {
    // ================================ producer: lane = aggregation ====================================
    uint32_t cur = 0xFFFFFFFFu, n_aggs = 0, num_docs = 0, bits = 0;
    const uint8_t* src0 = nullptr;
    for (uint32_t work = w_begin, seq = 0; work < w_end; work++, seq++) {
      while (__ldg(p.wl.first_work + split + 1) <= work) split++;
      if (split != cur) {
        cur = split;
        const DSplitPlan& P = p.plans[split];
        n_aggs = P.n_aggs; num_docs = P.num_docs; bits = 0;
        if (lane < n_aggs) {
          const DCol& c = p.cols[P.col_base + p.aggs[P.agg_base + lane].col];
          bits = c.bits;
          src0 = (const uint8_t*)P.data_base + c.values_off;
        }
      }
      const uint32_t d0 = (work - __ldg(p.wl.first_work + split)) * QA_CHUNK;
      const uint32_t nd = min((uint32_t)QA_CHUNK, num_docs - d0);
      const uint32_t slot = seq % QA_SLOTS;
      mbar_wait(bar_empty(slot), ((seq / QA_SLOTS) & 1u) ^ 1u);
      const uint32_t sl = sm.slot0 + slot * sm.slot_stride;
      const uint32_t bytes = (uint32_t)(((uint64_t)nd * bits + 127) >> 7) << 4;  // whole 16-byte words (the array is padded)
      uint32_t total = bytes;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(QW_FULL, total, o);
      if (lane == 0) {
        *(uint4*)(qw_smem + sl + sm.hdr) = make_uint4(split, d0, nd, 0u);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_full(slot)), "r"(total) : "memory");
      }
      __syncwarp();
      if (bytes) bulk_g2s(sbase + sl + sm.col_off[lane & (QA_MAX_AGGS - 1)], src0 + ((uint64_t)d0 * bits >> 3), bytes, bar_full(slot));
    }
  } else {
    // ================================ consumers =====================================================
    uint32_t cur_split = 0xFFFFFFFFu, n_aggs = 0;
    unsigned long long my_docs = 0;  // thread 0 counts the docs of the current split
    uint4* bcache = (uint4*)(qw_smem + sm.bcache) + warp * QA_MAX_AGGS;  // {lo, hi, bucket, valid} per aggregation
    auto enter_split = [&](uint32_t next) {
      // all consumer warps have added their counts of the old split: named barrier over the consumers
      asm volatile("bar.sync 1, %0;" ::"n"(QA_CW * 32) : "memory");
      if (cur_split != 0xFFFFFFFFu) {
        const DSplitPlan& P = p.plans[cur_split];
        QwAggCell* out = (QwAggCell*)P.out_cells;
        for (uint32_t i = tid; i < P.n_cells; i += QA_CW * 32) {
          const uint32_t v = cells[i];
          if (v) atomicAdd((unsigned long long*)&out[i].count, (unsigned long long)v);
        }
        if (tid == 0) flush_counts(P, P.sa.present, P.max_hits, my_docs, 0);
      }
      my_docs = 0;
      cur_split = next;
      if (next != 0xFFFFFFFFu) {
        const DSplitPlan& P = p.plans[next];
        n_aggs = P.n_aggs;
        for (uint32_t i = tid; i < P.n_cells; i += QA_CW * 32) cells[i] = 0;
        if (tid < n_aggs) {
          const DAgg& a = p.aggs[P.agg_base + tid];
          AggRow r;
          r.kind = a.kind; r.bits = p.cols[P.col_base + a.col].bits; r.cell_base = a.cell_base; r.nb = a.num_buckets;
          r.inv_step = a.inv_step; r.pad = 0; r.bounds = a.bounds; r.b0 = 0; r.bn = 0;
          if (a.kind == QW_AGG_HISTOGRAM) { r.b0 = __ldg((const uint64_t*)a.bounds); r.bn = __ldg((const uint64_t*)a.bounds + a.num_buckets); }
          atab[tid] = r;
        }
        if (lane < QA_MAX_AGGS) bcache[lane] = make_uint4(1u, 0u, 0u, 0u);  // empty interval: lo > hi
      }
      asm volatile("bar.sync 1, %0;" ::"n"(QA_CW * 32) : "memory");
    };
    for (uint32_t work = w_begin, seq = 0; work < w_end; work++, seq++) {
      const uint32_t slot = seq % QA_SLOTS;
      mbar_wait(bar_full(slot), (seq / QA_SLOTS) & 1u);
      const uint32_t sl = sm.slot0 + slot * sm.slot_stride;
      const uint4 h = *(const uint4*)(qw_smem + sl + sm.hdr);
      if (h.x != cur_split) enter_split(h.x);
      const uint32_t nd = h.z;
      if (tid == 0) my_docs += nd;
      const uint32_t g = tid;                                     // this thread's group of the chunk
      const uint32_t gv = nd > 32u * g ? min(32u, nd - 32u * g) : 0u;  // docs of the group that exist
      const bool warp_full = nd >= 32u * (tid | 31u) + 32u;            // all 32 groups of this warp are whole
      for (uint32_t gi = 0; gi < n_aggs; gi++) {
        const uint4 r0 = *(const uint4*)&atab[gi];  // kind, bits, cell_base, nb
        const uint32_t bits = r0.y;
        const uint32_t* w = (const uint32_t*)(qw_smem + sl + sm.col_off[gi]) + g * bits;
        uint32_t* ctr = cells + r0.z;
        if (r0.x == QW_AGG_HISTOGRAM) {
          uint32_t mn = 0xFFFFFFFFu, mx = 0;
          if (bits == 0) mn = 0;
          else if (gv == 32u) {
            uint32_t px = 0;
            unpack32_dyn(bits, w, [&](int v, uint32_t x) {
              if (v & 1) { mn = __vimin3_u32(mn, px, x); mx = __vimax3_u32(mx, px, x); } else px = x;
            });
          }
          // the warp's 1024 docs against the bucket the warp was in last time (time-ordered logs stay in
          // a bucket for many chunks): two warp reductions and two compares instead of two table searches
          const uint4 bc = bcache[gi];
          if (warp_full && __reduce_min_sync(QW_FULL, mn) >= bc.x && __reduce_max_sync(QW_FULL, mx) <= bc.y) {
            if (lane == 0) atomicAdd(&ctr[bc.z], 1024u);
            continue;
          }
          const AggRow& row = atab[gi];
          const uint64_t* B = (const uint64_t*)row.bounds;
          uint32_t bk_lo = 0, bk_hi = 1;
          const bool whole = gv == 32u && hist_bucket(B, r0.w, row.inv_step, row.b0, row.bn, mn, bk_lo) &&
                             hist_bucket(B, r0.w, row.inv_step, row.b0, row.bn, mx, bk_hi) && bk_lo == bk_hi;
          if (whole) atomicAdd(&ctr[bk_lo], 32u);
          else if (gv) {
            // the group straddles a bucket boundary / the hard bounds, or is the split's last: per doc
            for (uint32_t v = 0; v < gv; v++) {
              uint32_t x = 0;
              if (bits) {
                const uint32_t bp = v * bits, sh = bp & 31u;
                x = __funnelshift_r(w[bp >> 5], w[(bp >> 5) + 1], sh) & __funnelshift_lc(0xFFFFFFFFu, 0u, bits);
              }
              uint32_t bk;
              if (hist_bucket(B, r0.w, row.inv_step, row.b0, row.bn, x, bk)) atomicAdd(&ctr[bk], 1u);
            }
          }
          // remember the bucket of the warp's last whole group: raws in [B[bk], B[bk + 1]) (32-bit raws)
          const uint32_t wm = __ballot_sync(QW_FULL, whole);
          if (wm) {
            const uint32_t src = 31u - __clz(wm);
            const uint32_t bk = __shfl_sync(QW_FULL, bk_lo, src);
            if (lane == 0) {
              const uint64_t lo = __ldg(B + bk), hi = __ldg(B + bk + 1) - 1;
              bcache[gi] = make_uint4((uint32_t)lo, hi > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)hi, bk, 1u);
            }
          }
          __syncwarp();
        } else {
          // TERMS: dense index = raw value (ordinal of a string column)
          if (bits == 0) {
            if (gv) atomicAdd(&ctr[0], gv);
          } else if (bits <= 2) {
            // bit planes: 32 docs per popcount. Plane bit positions: value v < 16 -> bit 2v, v >= 16 -> bit 2(v-16)+1
            // (1-bit columns: value v -> bit v); `vm` = the positions of the docs that exist
            uint32_t lo, hi, vm;
            if (bits == 1) {
              lo = gv ? w[0] : 0u; hi = 0;
              vm = gv >= 32u ? 0xFFFFFFFFu : ((1u << gv) - 1u);
            } else {
              const uint32_t a0 = gv ? w[0] : 0u, a1 = gv > 16u ? w[1] : 0u;
              lo = (a0 & 0x55555555u) | ((a1 & 0x55555555u) << 1);
              hi = ((a0 >> 1) & 0x55555555u) | (a1 & 0xAAAAAAAAu);
              const uint32_t n0 = min(gv, 16u), n1 = gv > 16u ? gv - 16u : 0u;
              const uint32_t m0 = n0 >= 16u ? 0x55555555u : (((1u << (2u * n0)) - 1u) & 0x55555555u);
              const uint32_t m1 = n1 >= 16u ? 0x55555555u : (((1u << (2u * n1)) - 1u) & 0x55555555u);
              vm = m0 | (m1 << 1);
            }
            lo &= vm; hi &= vm;
            const uint32_t t3 = __popc(lo & hi), t1 = __popc(lo) - t3, t2 = __popc(hi) - t3, t0 = __popc(vm) - t1 - t2 - t3;
            // warp totals (all 32 lanes are here: the branch is uniform): each count is <= 32, so the four
            // fit one 32-bit word as 8-bit fields x 32 lanes = 10-bit sums -> two packed reductions
            const uint32_t s01 = __reduce_add_sync(QW_FULL, t0 | (t1 << 16)), s23 = __reduce_add_sync(QW_FULL, t2 | (t3 << 16));
            if (lane == 0) {
              if (s01 & 0xFFFFu) atomicAdd(&ctr[0], s01 & 0xFFFFu);
              if (s01 >> 16) atomicAdd(&ctr[1], s01 >> 16);
              if (s23 & 0xFFFFu) atomicAdd(&ctr[2], s23 & 0xFFFFu);
              if (s23 >> 16) atomicAdd(&ctr[3], s23 >> 16);
            }
          } else {
            for (uint32_t v = 0; v < gv; v++) {
              const uint32_t bp = v * bits, sh = bp & 31u;
              const uint32_t x = __funnelshift_r(w[bp >> 5], w[(bp >> 5) + 1], sh) & __funnelshift_lc(0xFFFFFFFFu, 0u, bits);
              atomicAdd(&ctr[x], 1u);
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty(slot));
    }
    enter_split(0xFFFFFFFFu);
  }
}

}  // namespace qwk
