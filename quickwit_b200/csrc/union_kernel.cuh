// union_kernel.cuh — the BM25 top-K shape (pure OR of positive-weight scored terms ranked by _score)
// as a warp-specialised TMA + mbarrier pipeline for sm_90a (Hopper).
//
// Replaces tantivy's BufferedUnionScorer + Bm25Weight + TopDocs loop behind `searcher.search`
// (quickwit-search/src/leaf.rs:637; SURVEY.md §8a rows a3-a5, a10-a11) for the headline query shape.
//
// One 448-thread block = 13 consumer warps + 1 producer warp, two blocks per SM. The block owns one
// 16384-doc window of one split at a time (f32 score accumulator of the window in shared memory);
// each block walks its own contiguous chunk of the flat (split, window) list.
//
//   producer warp   per window: (1) lane = term: one load of the term's window-index entry (QwWinIdx)
//                   gives the ordinals of the posting blocks overlapping the window; (2) lane = block:
//                   a coalesced 16-byte load of the block's skip entry (QwSkip) tells its widths and
//                   doc range; blocks that miss the window are dropped; the survivors are packed into
//                   the current pipeline slot — one `cp.async.bulk` (1-D TMA) per block straight from
//                   HBM to shared memory, completion counted on the slot's `full` mbarrier — and
//                   described by a 16-byte record (shared address, widths, clause, interior flag).
//                   A slot that fills up is closed and the window continues in the next slot, so any
//                   density / term count works. No consumer ever executes a staging instruction.
//   consumer warps  wait on `full`, take blocks round-robin, decode one block per warp (4-lane-
//                   interleaved bit-unpack -> warp-shuffle prefix scan -> doc ids; tf unpack; the
//                   per-posting fieldnorm id comes with the block, so BM25 = weight * tff[tf][fn] is
//                   one PRMT + one table load per posting) and add the four contributions per lane
//                   into the score array.
//   clause order    f32 sums must follow the reference's clause order. Every clause of a window is a
//                   STAGE of a per-block ring of mbarriers ("chain", one arrival per consumer warp
//                   per stage): a warp arrives at a stage when it has no more blocks in it and waits
//                   for stage s-1 before it touches the accumulator for stage s. Decode never waits,
//                   only the read-modify-write does; there is no __syncthreads, no spin on shared
//                   memory and no fence in the loop. The sweep of a finished window (count matches,
//                   threshold test, clear) is one more stage of the same chain, so the next window's
//                   decode overlaps the sweep of this one.
//   own sample      MODE_SAMPLE_COLLECT: each block's first window is its share of the threshold sample; the
//                   blocks meet at a grid barrier (cooperative launch), pick the threshold from the complete
//                   histogram, sweep the first window against it, and collect the rest as MODE_COLLECT does.
#pragma once
#include "kernels.cuh"

namespace qwk {

/* 13 consumer warps + the producer, two blocks per SM: 72 registers per thread (sm_90a: 40 B of spill stores in the
 * COLLECT instantiation, 36 B in SAMPLE_COLLECT). Measured on one H100 80GB HBM3 (400 W power limit), k_union<COLLECT> per launch on the bench
 * workload: 201-202 us; 384 threads / 80 registers (56 B of spills): 204-205 us; 512 threads / 64 registers (292 B of
 * spills): 211-213 us. */
#define QU_THREADS 448
#define QU_NCW (QU_THREADS / 32 - 1)   /* consumer warps; warp QU_NCW is the producer */
#define QU_NCT (QU_NCW * 32)
#define QU_SLOTS 2
#define QU_MAXBLK 128           /* block records per slot */
#define QU_CHAIN 128            /* mbarriers in the stage ring (a warp is never > 70 stages ahead) */
#define QU_MAX_TERMS 32
#define QU_SUSPEND_NS 100000u   /* try_wait suspend-time hint: a waiting warp sleeps in hardware instead of polling */
#define QU_PAD 32               /* decode may read one 16-byte word past a block */
#define QU_CANDS 16             /* per-warp buffer of docs that reached the score lower bound */
#define QU_MINB 2               /* blocks per SM */

enum { QU_F_FIRST = 1u, QU_F_LAST = 2u, QU_F_END = 4u };

struct USmem {
  uint32_t score;                       // float[W]
  uint32_t slot0, slot_stride;          // QU_SLOTS slots
  uint32_t payload, recs, ttab, hdr;    // offsets inside a slot
  uint32_t bars;                        // full[QU_SLOTS], empty[QU_SLOTS], chain[QU_CHAIN]
  uint32_t hist;                        // MODE_HIST: uint32[QW_HIST_BINS]
  uint32_t cands;                       // uint2[QU_NCW][QU_CANDS], then uint32 count[QU_NCW]
  uint32_t thr;                         // MODE_SAMPLE_COLLECT: DThresh[2], then uint32 split[2] (the chunk's splits)
  uint32_t cap;                         // payload bytes per slot
  uint32_t total;
};

struct UParams {
  const DSplitPlan* plans;
  const DInstr* instrs;
  const DCol* cols;
  DThresh* thresh;             // COLLECT: read; SAMPLE_COLLECT: written for the host by each split's first block
  DWorkList wl;                   // (split, window) list; sampled passes: the sampled windows
  const uint32_t* sample_stride;  // SAMPLE_COLLECT: per split, the weight of its sample (qw_fused_sample_plan)
  uint32_t* sync;                 // SAMPLE_COLLECT: grid barrier counter, zero at launch
  uint32_t* err;                  // SAMPLE_COLLECT: set to 1 when the grid barrier timed out
  uint32_t W;
  USmem sm;
};

struct UHdr {  // 32 bytes, written by the producer when it closes a slot
  uint32_t ws, wlen, split, flags;
  uint32_t n_blocks, n_terms, t_last;  // t_last: clause of the slot's last block (stages below it are final)
  float s_lo;                          // COLLECT: f32 lower bound of the threshold bucket; HIST: score_scale (unused in SAMPLE_COLLECT)
};

// level-0 digit of a score's composite key: [1 | lin:10] (score_lin)
__device__ __forceinline__ uint32_t score_digit(float s, float scale) {
  const float x = __fmul_rn(s, scale);
  const uint32_t l = x >= 1023.0f ? 1023u : (x > 0.0f ? (uint32_t)x : 0u);
  return 1024u | l;
}

// f32 lower bound of a threshold's level-0 score bucket (conservative: one part in 2^20); -1: no threshold
__device__ __forceinline__ float thresh_s_lo(const DThresh& T, float score_scale) {
  const uint32_t thr_top = (uint32_t)(T.key[0] >> 53);
  return thr_top >= 1024u ? __fmul_rn(__fdiv_rn((float)(thr_top & 1023u), score_scale), 0.999999f) : -1.0f;
}

__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Grid-wide barrier of k_union<MODE_SAMPLE_COLLECT>, called by one thread per block after the block's consumer warps
// have met (so the fence below orders their global atomics before the arrival). False when the other blocks did not
// all arrive within a second: the caller reports it, and the kernel still ends normally.
//
// Safe only because the kernel is launched cooperatively (cudaLaunchCooperativeKernel), with a grid of at most
// occupancy x SM count blocks. The CUDA Programming Guide, on grid synchronization: "To guarantee the co-residency of
// the thread blocks on the GPU, the number of blocks launched needs to be carefully considered." The runtime API
// (cudaLaunchCooperativeKernel): "The total number of blocks launched cannot exceed the maximum number of blocks per
// multiprocessor as returned by cudaOccupancyMaxActiveBlocksPerMultiprocessor (or
// cudaOccupancyMaxActiveBlocksPerMultiprocessorWithFlags) times the number of multiprocessors as specified by the
// device attribute cudaDevAttrMultiProcessorCount." A grid launched that way has all of its blocks resident together,
// also while other calls' kernels run on other streams, so no block waits here for one that cannot start.
__device__ __forceinline__ bool grid_barrier(uint32_t* ctr, uint32_t n_blocks) {
  __threadfence();
  atomicAdd(ctr, 1u);
  const uint64_t t0 = globaltimer_ns();
  for (;;) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
    if (v >= n_blocks) break;
    if (globaltimer_ns() - t0 > 1000000000ull) return false;
    __nanosleep(500);
  }
  __threadfence();
  return true;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.expect_tx.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1, %2;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}" ::"r"(bar), "r"(parity), "r"(QU_SUSPEND_NS) : "memory");
}
// 1-D TMA: global -> shared, completion (bytes) on an mbarrier of this block
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(__cvta_generic_to_global(src)), "r"(bytes), "r"(bar)
               : "memory");
}
// inclusive scan step over segments of `1 << LOGW` lanes, with the shuffle's own predicate
// (SHFL.UP + predicated IADD)
template <int LOGW>
__device__ __forceinline__ uint32_t scan_step(uint32_t x, uint32_t o) {
  constexpr uint32_t c = (32u - (1u << LOGW)) << 8;
  asm volatile("{\n.reg .u32 t;\n.reg .pred p;\nshfl.sync.up.b32 t|p, %0, %1, %2, 0xffffffff;\n@p add.u32 %0, %0, t;\n}" : "+r"(x) : "r"(o), "n"(c));
  return x;
}
__device__ __forceinline__ uint32_t seg16_incl_scan(uint32_t x) {
  x = scan_step<4>(x, 1); x = scan_step<4>(x, 2); x = scan_step<4>(x, 4); x = scan_step<4>(x, 8);
  return x;
}
__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t x) {
  x = scan_step<5>(x, 1); x = scan_step<5>(x, 2); x = scan_step<5>(x, 4); x = scan_step<5>(x, 8); x = scan_step<5>(x, 16);
  return x;
}

// Rare path of the sweep: a doc that reaches the float lower bound builds its composite key and, if
// it reaches the threshold key, joins the split's candidate list (k_select sorts it out).
__device__ __noinline__ void union_emit(const DSplitPlan* plans, const DThresh& T, const DCol* cols, uint32_t split, uint32_t doc, float sc) {
  const DSplitPlan& P = plans[split];
  const Key thr{T.key[0], T.key[1], T.key[2]};
  const DocKey dk = doc_key(P, P.key, cols + P.col_base, (const uint8_t*)P.data_base, doc, sc);
  if (key_ge(dk.key, thr)) push_cand(P, dk.key);
}

template <int MODE>
__global__ void __launch_bounds__(QU_THREADS, QU_MINB) k_union(const UParams p) {
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t W = p.W;
  const uint32_t sbase = smem_u32(qw_smem);
  const uint32_t bars = sbase + p.sm.bars;
  auto bar_full = [&](uint32_t s) { return bars + 8u * s; };
  auto bar_empty = [&](uint32_t s) { return bars + 8u * (QU_SLOTS + s); };
  auto bar_chain = [&](uint32_t st) { return bars + 8u * (2 * QU_SLOTS + (st & (QU_CHAIN - 1))); };
  auto chain_parity = [&](uint32_t st) { return (st / QU_CHAIN) & 1u; };
  if (tid == 0) {
    for (uint32_t s = 0; s < QU_SLOTS; s++) { mbar_init(bar_full(s), 1); mbar_init(bar_empty(s), QU_NCW); }
    for (uint32_t s = 0; s < QU_CHAIN; s++) mbar_init(bar_chain(s), QU_NCW);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  // this block's chunk of the flat (split, window) list (handing windows out one at a time from a global counter was
  // slower: consecutive windows of a block then belong to different splits, and the plan switch sits on the
  // producer's critical path)
  const uint32_t w_begin = qw_chunk_begin(p.wl.total_work, blockIdx.x, gridDim.x);
  const uint32_t w_end = qw_chunk_begin(p.wl.total_work, blockIdx.x + 1, gridDim.x);

  if (warp == QU_NCW) {
    // ================================ producer ======================================================
    uint32_t seq = 0;            // slots closed so far
    uint32_t cur_split = 0;
    // lane = term slot of the current split's plan
    uint64_t t_data = 0, t_widx = 0, t_skip = 0, t_tab = 0;
    uint32_t t_nblk = 0, t_shift = 0, t_fl = 0, t_sub16 = 0;
    float t_w = 0.f;
    const uint8_t* base = nullptr;
    uint32_t n_terms = 0, num_docs = 0;
    float hdr_f = -1.0f;
    // slot state (warp-uniform)
    bool open = false;
    uint32_t slot = 0, off = 0, cnt = 0, last_t = 0, last_t_l = 0;
    bool first_of_window = true;
    uint32_t ws = 0, wlen = 0;
    auto slot_base = [&](uint32_t s) { return p.sm.slot0 + s * p.sm.slot_stride; };
    auto open_slot = [&]() {
      slot = seq % QU_SLOTS;
      mbar_wait(bar_empty(slot), ((seq / QU_SLOTS) & 1u) ^ 1u);
      open = true; off = 0; cnt = 0;
      if (lane == 0) *(uint32_t*)(qw_smem + slot_base(slot) + p.sm.hdr + 32) = 0;  // next block to hand out
      if (lane < n_terms) {
        uint4 tt;
        tt.x = __float_as_uint(t_w); tt.y = t_fl; tt.z = (uint32_t)t_tab; tt.w = (uint32_t)(t_tab >> 32);
        *(uint4*)(qw_smem + slot_base(slot) + p.sm.ttab + 16u * lane) = tt;
      }
    };
    auto close_slot = [&](uint32_t flags) {
      if (lane == 0) {
        uint4* d = (uint4*)(qw_smem + slot_base(slot) + p.sm.hdr);
        d[0] = make_uint4(ws, wlen, cur_split, flags | (first_of_window ? QU_F_FIRST : 0u));
        d[1] = make_uint4(cnt, n_terms, last_t, __float_as_uint(hdr_f));
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_full(slot));
      seq++;
      open = false;
      first_of_window = false;
    };
    auto load_plan = [&](uint32_t split) {
      cur_split = split;
      const DSplitPlan& P = p.plans[split];
      base = (const uint8_t*)P.data_base;
      n_terms = P.n_terms;
      num_docs = P.num_docs;
      t_nblk = 0;
      if (lane < n_terms) {
        const DInstr& in = p.instrs[P.instr_base + 1 + lane];  // [BOOL_BEGIN, TERM x n, BOOL_END]
        t_data = in.a; t_widx = in.b; t_skip = in.c; t_nblk = in.n; t_shift = in.m;
        t_fl = in.flags; t_w = in.f; t_sub16 = in.pad;
        t_tab = P.bm25_tab[in.r];
      }
      // (SAMPLE_COLLECT: the consumers pick the threshold themselves, after the producer has moved on)
      if (MODE == MODE_COLLECT) hdr_f = thresh_s_lo(p.thresh[split], P.key.score_scale);
      else hdr_f = P.key.score_scale;
    };
    uint4 wa = make_uint4(0, 0, 0, 0), wb = wa;  // this lane's window-index entries (first / last index window)
    auto load_widx = [&](uint32_t window) {
      wa = wb = make_uint4(0, 0, 0, 0);
      const uint32_t s = window * W, e = min(s + W, num_docs);
      if (lane < n_terms && t_nblk) {
        const uint4* wi = (const uint4*)(base + t_widx);
        const uint32_t e0 = s >> t_shift, e1 = (e - 1) >> t_shift;
        wa = __ldg(wi + e0);
        wb = e1 != e0 ? __ldg(wi + e1) : wa;
      }
    };
    auto window_of = [&](uint32_t work, uint32_t split) {
      return qw_sample_item(work - __ldg(p.wl.first_work + split), split, p.wl.stride);
    };
    // split of a work item: number of prefix entries <= work, minus one (lane-parallel; empty splits share their entry)
    auto split_of = [&](uint32_t work) {
      uint32_t cnt = 0;
      for (uint32_t b0 = 0; b0 < p.wl.n_splits; b0 += 32) {
        const uint32_t i = b0 + lane;
        cnt += __popc(__ballot_sync(QW_FULL, i < p.wl.n_splits && __ldg(p.wl.first_work + i) <= work));
      }
      return cnt - 1;
    };
    uint32_t split = 0;
    uint32_t work = w_begin, next_work = w_begin + 1;
    if (work < w_end) {
      split = split_of(work);
      load_plan(split);
      load_widx(window_of(work, split));
    }
    for (; work < w_end; ) {
      const uint32_t window = window_of(work, split);
      ws = window * W;
      const uint32_t we = min(ws + W, num_docs);
      wlen = we - ws;
      first_of_window = true;
      // ---- lane = term: blocks of the term that overlap the window (entries loaded one window ago) --
      const uint32_t fb = wa.z;
      const uint32_t nb = (wb.y > wa.x && wb.w > wa.z) ? wb.w - wa.z : 0;
      const uint32_t incl_nb = warp_incl_scan(nb);
      const uint32_t gbase = incl_nb - nb;
      const uint32_t G = __shfl_sync(QW_FULL, incl_nb, 31);
      // ---- lane = block: skip + checkpoint entries -> record, runs of blocks -> bulk copies ----------
      auto round_loads = [&](uint32_t q0, uint32_t& t_out, uint4& r_out, uint4& c_out, uint64_t& dat_out, uint32_t& tfl_out) {
        const uint32_t q = q0 + lane;
        uint32_t t = 0;  // clause of flat block q: the last term slot whose first block is <= q
#pragma unroll
        for (uint32_t step = 16; step; step >>= 1) {
          const uint32_t cand = t + step;
          const uint32_t gb = __shfl_sync(QW_FULL, gbase, cand & 31);
          if (cand < 32 && gb <= q) t = cand;
        }
        const uint32_t k = q - __shfl_sync(QW_FULL, gbase, t);
        const uint32_t fbt = __shfl_sync(QW_FULL, fb, t);
        const uint64_t skp = __shfl_sync(QW_FULL, t_skip, t);
        const uint32_t sub16 = __shfl_sync(QW_FULL, t_sub16, t);
        dat_out = __shfl_sync(QW_FULL, t_data, t);
        tfl_out = __shfl_sync(QW_FULL, t_fl, t);
        r_out = c_out = make_uint4(0, 0, 0, 0);
        if (q < G) r_out = __ldg((const uint4*)(base + skp) + fbt + k);  // last_doc, prev_last_doc, byte_off, widths/count
        (void)sub16;
        t_out = t;
      };
      uint32_t t = 0, tfl = 0;
      uint4 r = make_uint4(0, 0, 0, 0), ck = r;
      uint64_t dat = 0;
      if (G) round_loads(0, t, r, ck, dat, tfl);
      // the next window's index entries fly while this window is packed (same split: same term constants)
      uint32_t nx_split = split;
      const bool have_next = next_work < w_end;
      if (have_next) {
        while (__ldg(p.wl.first_work + nx_split + 1) <= next_work) nx_split++;
        if (nx_split == split) load_widx(window_of(next_work, split));
      }
      for (uint32_t q0 = 0; q0 < G; q0 += 32) {
        const uint32_t q = q0 + lane;
        uint32_t t2 = 0, tfl2 = 0;
        uint4 r2 = make_uint4(0, 0, 0, 0), ck2 = r2;
        uint64_t dat2 = 0;
        if (q0 + 32 < G) round_loads(q0 + 32, t2, r2, ck2, dat2, tfl2);  // next round's loads fly during this round
        const uint32_t doc_bits = r.w & 0xFF, tf_bits = (r.w >> 8) & 0xFF;
        const uint32_t first_lb = r.y + 1;  // lower bound of the first doc (0 when prev == 0xFFFFFFFF)
        const bool overlaps = q < G && r.x >= ws && first_lb < we;
        // bytes of the block in the image: inline header + packed docs + packed tfs + fieldnorm ids
        const uint32_t size = overlaps ? 16u + 16u * (doc_bits + tf_bits) + ((tfl & IF_HAS_FN) ? QW_BLOCK_LEN : 0u) : 0u;
        const uint8_t* src = base + dat + r.z;
        uint32_t pending = __ballot_sync(QW_FULL, overlaps);
        while (pending) {
          if (!open) open_slot();
          const bool mine = (pending >> lane) & 1u;
          const uint32_t sz = mine ? size : 0u;
          const uint32_t incl = warp_incl_scan(sz);
          const uint32_t pos = __popc(pending & ((1u << lane) - 1u));
          const bool fits = mine && off + incl <= p.sm.cap && cnt + pos < QU_MAXBLK;
          const uint32_t fitmask = __ballot_sync(QW_FULL, fits);  // a prefix of `pending`
          if (fitmask) {
            const uint32_t lastfit = 31u - __clz(fitmask);
            const uint32_t bytes = __shfl_sync(QW_FULL, incl, lastfit);
            if (lane == 0) mbar_expect_tx(bar_full(slot), bytes);
            __syncwarp();
            // a run = consecutive fitting lanes of one term: its blocks are contiguous in the image
            const uint32_t t_prev = __shfl_up_sync(QW_FULL, t, 1);
            const bool head = fits && (lane == 0 || !((fitmask >> (lane - 1)) & 1u) || t_prev != t);
            const uint32_t heads = __ballot_sync(QW_FULL, head);
            const uint32_t above = lane == 31 ? 0u : (heads & ~((2u << lane) - 1u));  // run heads after this lane
            const uint32_t last = above ? (uint32_t)__ffs(above) - 2u : lastfit;      // last lane of this lane's run (heads only)
            const uint32_t run_end = __shfl_sync(QW_FULL, incl, last & 31u);
            const uint32_t dst = sbase + slot_base(slot) + p.sm.payload + off + incl - sz;
            if (fits) {
              const bool interior = first_lb >= ws && r.x < we && (r.w >> 16) == QW_BLOCK_LEN;
              *(uint4*)(qw_smem + slot_base(slot) + p.sm.recs + 16u * (cnt + pos)) = make_uint4(r.y, dst + 16u, r.w, t | (interior ? 256u : 0u));
              last_t_l = t;
            }
            if (head) bulk_g2s(dst, src, run_end - (incl - sz), bar_full(slot));
            off += bytes;
            cnt += __popc(fitmask);
            last_t = __shfl_sync(QW_FULL, last_t_l, lastfit);
            pending &= ~fitmask;
          }
          if (pending) close_slot(0);  // slot full: the window continues in the next slot
        }
        t = t2; tfl = tfl2; r = r2; ck = ck2; dat = dat2;
      }
      // (the sample window reaches the consumers even without a block: they meet the other blocks after it)
      if (MODE == MODE_SAMPLE_COLLECT && !open && work == w_begin) open_slot();
      if (open) close_slot(QU_F_LAST);
      if (have_next && nx_split != split) {
        split = nx_split;
        load_plan(split);
        load_widx(window_of(next_work, split));
      }
      work = next_work;
      next_work = work + 1;
    }
    // terminal slot
    open_slot();
    cnt = 0;
    close_slot(QU_F_END);
  } else {
    // ================================ consumers =====================================================
    float* score = (float*)(qw_smem + p.sm.score);
    uint32_t* hist = (uint32_t*)(qw_smem + p.sm.hist);
    {
      float4* q = reinterpret_cast<float4*>(score);
      for (uint32_t i = tid; i < (W >> 2); i += QU_NCT) q[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (MODE == MODE_HIST) for (uint32_t i = tid; i < QW_HIST_BINS; i += QU_NCT) hist[i] = 0;
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_chain(0));
    uint32_t my_stage = 1;   // stages this warp has arrived at: [0, my_stage)
    uint32_t waited = 0;     // stages known complete: [0, waited)
    uint32_t wbase = 1;      // stage of clause 0 of the current window
    uint32_t next_base = 1;
    uint32_t cur_split = 0xFFFFFFFFu;
    uint32_t my_hits = 0;
    uint2* cands = (uint2*)(qw_smem + p.sm.cands) + warp * QU_CANDS;
    uint32_t* ncand = (uint32_t*)(qw_smem + p.sm.cands + QU_NCW * QU_CANDS * 8) + warp;
    if (lane == 0) *ncand = 0;
    // SAMPLE_COLLECT: the thresholds of the chunk's (one or two) splits, picked by the block itself
    DThresh* s_thr = (DThresh*)(qw_smem + p.sm.thr);
    uint32_t* s_thr_split = (uint32_t*)(s_thr + 2);
    float* s_thr_lo = (float*)(s_thr_split + 2);
    auto thr_of = [&](uint32_t split) -> const DThresh& {
      if (MODE == MODE_SAMPLE_COLLECT) return s_thr[split == s_thr_split[0] ? 0 : 1];
      return p.thresh[split];
    };
    auto pass_to = [&](uint32_t st) {  // arrive at every stage below st
      if (my_stage < st) {
        __syncwarp();
        // one lane per stage (a warp that skips several clauses arrives at all of them with one instruction)
        for (uint32_t s0 = my_stage; s0 < st; s0 += 32) if (s0 + lane < st) mbar_arrive(bar_chain(s0 + lane));
        my_stage = st;
      }
    };
    auto wait_below = [&](uint32_t st) {  // all stages below st complete
      if (waited < st) {
        mbar_wait(bar_chain(st - 1), chain_parity(st - 1));
        waited = st;
      }
    };
    // candidates -> composite key -> the split's candidate list (k_select sorts it out); lane-parallel
    auto flush_cands = [&]() {
      __syncwarp();
      const uint32_t n = min(*ncand, (uint32_t)QU_CANDS);
      if (n == 0) return;
      const DSplitPlan& P = p.plans[cur_split];
      const DThresh& T = thr_of(cur_split);
      const Key thr{T.key[0], T.key[1], T.key[2]};
      bool pass = false;
      DocKey dk;
      dk.key = Key{0, 0, 0};
      if (lane < n) {
        const uint2 c = cands[lane];
        dk = doc_key(P, P.key, p.cols + P.col_base, (const uint8_t*)P.data_base, c.x, __uint_as_float(c.y));
        pass = key_ge(dk.key, thr);
      }
      const uint32_t m = __ballot_sync(QW_FULL, pass);
      if (m) {
        uint32_t basepos = 0;
        if (lane == 0) basepos = atomicAdd((uint32_t*)P.out_cand_count, (uint32_t)__popc(m));
        basepos = __shfl_sync(QW_FULL, basepos, 0);
        const uint32_t pos = basepos + __popc(m & ((1u << lane) - 1u));
        if (pass && pos < qw_cand_cap(P.max_hits)) {
          uint64_t* c = (uint64_t*)P.out_cands + 3ull * pos;
          c[0] = dk.key.w0; c[1] = dk.key.w1; c[2] = dk.key.w2;
        }
      }
      __syncwarp();
      if (lane == 0) *ncand = 0;
      __syncwarp();
    };
    auto flush_hits = [&]() {
      if (MODE == MODE_HIST || cur_split == 0xFFFFFFFFu) return;
      flush_cands();
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) my_hits += __shfl_down_sync(QW_FULL, my_hits, o);
      if (lane == 0 && my_hits) {
        const DSplitPlan& P = p.plans[cur_split];
        flush_counts(P, P.sa.present, P.max_hits, my_hits, 0);
      }
      my_hits = 0;
    };

    auto collect_sweep = [&](const uint32_t ws, const uint32_t split, const float s_lo, const uint32_t end_stage) {
      wait_below(end_stage);  // every contribution of the window is in
      float4* sc4 = reinterpret_cast<float4*>(score);
      const uint32_t s_lo_bits = s_lo > 0.0f ? __float_as_uint(s_lo) : 1u;  // no threshold yet: every match goes on
#pragma unroll 4
      for (uint32_t q = tid; q < (W >> 2); q += QU_NCT) {
        const float4 v = sc4[q];
        sc4[q] = make_float4(0.f, 0.f, 0.f, 0.f);
        const float vv[4] = {v.x, v.y, v.z, v.w};
        // (scores are sums of positive contributions: as integers, 0 = no match and the order is the float order)
        const uint32_t u0 = __float_as_uint(vv[0]), u1 = __float_as_uint(vv[1]), u2 = __float_as_uint(vv[2]), u3 = __float_as_uint(vv[3]);
        my_hits += min(u0, 1u) + min(u1, 1u) + min(u2, 1u) + min(u3, 1u);
        if (__vimax3_u32(__vimax3_u32(u0, u1, u2), u3, 0u) >= s_lo_bits) {
#pragma unroll
          for (int j = 0; j < 4; j++) {
            if (vv[j] > 0.0f && vv[j] >= s_lo) {
              const uint32_t pos = atomicAdd(ncand, 1u);
              if (pos < QU_CANDS) cands[pos] = make_uint2(ws + 4 * q + j, __float_as_uint(vv[j]));
              else union_emit(p.plans, thr_of(split), p.cols, split, ws + 4 * q + j, vv[j]);  // buffer full: slow road now
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_chain(end_stage));
      my_stage = end_stage + 1;
      if (*ncand >= QU_CANDS / 2) flush_cands();  // (after the arrival: nobody waits for the global atomics)
    };

    for (uint32_t seq = 0;; seq++) {
      const uint32_t slot = seq % QU_SLOTS;
      mbar_wait(bar_full(slot), (seq / QU_SLOTS) & 1u);
      const uint32_t sl = p.sm.slot0 + slot * p.sm.slot_stride;
      const uint4 h0 = *(const uint4*)(qw_smem + sl + p.sm.hdr);
      const uint4 h1 = *(const uint4*)(qw_smem + sl + p.sm.hdr + 16);
      const uint32_t ws = h0.x, wlen = h0.y, split = h0.z, flags = h0.w;
      const uint32_t G = h1.x, n_terms = h1.y, t_last = h1.z;
      const float hdr_f = __uint_as_float(h1.w);
      if (flags & QU_F_END) break;
      if (flags & QU_F_FIRST) wbase = next_base;
      if (split != cur_split) {
        flush_hits();
        cur_split = split;
      }
      const uint32_t recs = sl + p.sm.recs, ttab = sl + p.sm.ttab;

      // Two blocks per warp step: half-warp `half` decodes block g0 + half, 16 lanes x 8 postings each (two
      // positions of the 4-lane-interleaved words per lane) — fewer warp instructions per block than a
      // 32 x 4 split, a 4-step scan, and eight independent postings per lane for the scheduler to overlap.
      const uint32_t half = lane >> 4, hl = lane & 15u;
      for (uint32_t g0 = 2u * warp; g0 < G; g0 += 2u * QU_NCW) {
        const bool on = g0 + half < G;
        const uint4 rec = *(const uint4*)(qw_smem + recs + 16u * (on ? g0 + half : g0));  // prev_last_doc, shared address, widths/count, clause | interior
        const uint32_t t = rec.w & 0xFFu;
        // This warp is done with every clause below the one it is about to decode: say so NOW, not after the
        // decode — the warps that wait for those stages are on the window's critical path (one hop per clause).
        const uint32_t st = wbase + t;
        const uint32_t st_lo = __shfl_sync(QW_FULL, st, 0);
        const uint32_t st_hi = __shfl_sync(QW_FULL, on ? st : 0u, 16);  // (0: the upper half has no block)
        pass_to(st_lo);
        const uint4 tt = *(const uint4*)(qw_smem + ttab + 16u * t);
        const float weight = __uint_as_float(tt.x);
        const float* tab = (const float*)(((uint64_t)tt.w << 32) | tt.z);
        const uint32_t blk = rec.y - sbase;  // offset inside qw_smem
        const uint32_t doc_bits = rec.z & 0xFFu, tf_bits = (rec.z >> 8) & 0xFFu;
        // ---- doc ids: two positions x 4 values per lane, in-lane prefix, then a 16-lane scan -------------
        // Both positions of a lane are adjacent in the packed stream: for widths <= 16 the 32 bits that start at
        // the first position hold the second one too, so ONE pair of 16-byte words serves both (half the
        // shared-memory loads of the general path).
        const bool narrow = __all_sync(QW_FULL, doc_bits <= 16u && tf_bits <= 16u);
        uint32_t d[8];
        if (narrow) {
          const uint32_t bp0 = 2u * hl * doc_bits;
          const uint8_t* a0 = qw_smem + blk + ((bp0 >> 5) << 4);
          const uint4 A0 = *(const uint4*)a0, B0 = *(const uint4*)(a0 + 16);
          const uint32_t sh0 = bp0 & 31u;
          const uint32_t mask = __funnelshift_lc(0xFFFFFFFFu, 0u, doc_bits);
          const uint32_t x0 = __funnelshift_r(A0.x, B0.x, sh0), x1 = __funnelshift_r(A0.y, B0.y, sh0);
          const uint32_t x2 = __funnelshift_r(A0.z, B0.z, sh0), x3 = __funnelshift_r(A0.w, B0.w, sh0);
          d[0] = (x0 & mask) + 1u;
          d[1] = d[0] + (x1 & mask) + 1u;
          d[2] = d[1] + (x2 & mask) + 1u;
          d[3] = d[2] + (x3 & mask) + 1u;
          d[4] = d[3] + ((x0 >> doc_bits) & mask) + 1u;
          d[5] = d[4] + ((x1 >> doc_bits) & mask) + 1u;
          d[6] = d[5] + ((x2 >> doc_bits) & mask) + 1u;
          d[7] = d[6] + ((x3 >> doc_bits) & mask) + 1u;
        } else {
          const uint32_t bp0 = 2u * hl * doc_bits, bp1 = bp0 + doc_bits;
          const uint8_t* a0 = qw_smem + blk + ((bp0 >> 5) << 4);
          const uint8_t* a1 = qw_smem + blk + ((bp1 >> 5) << 4);
          const uint4 A0 = *(const uint4*)a0, B0 = *(const uint4*)(a0 + 16);
          const uint4 A1 = *(const uint4*)a1, B1 = *(const uint4*)(a1 + 16);
          const uint32_t sh0 = bp0 & 31u, sh1 = bp1 & 31u;
          const uint32_t mask = __funnelshift_lc(0xFFFFFFFFu, 0u, doc_bits);
          // strictly-sorted deltas: doc[i] = doc[i-1] + v[i] + 1
          d[0] = (__funnelshift_r(A0.x, B0.x, sh0) & mask) + 1u;
          d[1] = d[0] + (__funnelshift_r(A0.y, B0.y, sh0) & mask) + 1u;
          d[2] = d[1] + (__funnelshift_r(A0.z, B0.z, sh0) & mask) + 1u;
          d[3] = d[2] + (__funnelshift_r(A0.w, B0.w, sh0) & mask) + 1u;
          d[4] = d[3] + (__funnelshift_r(A1.x, B1.x, sh1) & mask) + 1u;
          d[5] = d[4] + (__funnelshift_r(A1.y, B1.y, sh1) & mask) + 1u;
          d[6] = d[5] + (__funnelshift_r(A1.z, B1.z, sh1) & mask) + 1u;
          d[7] = d[6] + (__funnelshift_r(A1.w, B1.w, sh1) & mask) + 1u;
        }
        const uint32_t incl = seg16_incl_scan(d[7]);
        const uint32_t basev = rec.x + (incl - d[7]) - ws;  // mod 2^32; window-relative
        uint32_t r[8];
#pragma unroll
        for (int j = 0; j < 8; j++) r[j] = basev + d[j];
        // ---- term frequencies -----------------------------------------------------------------------
        uint32_t f[8];
#pragma unroll
        for (int j = 0; j < 8; j++) f[j] = 1;
        if (tf_bits && narrow) {
          const uint32_t bp0 = 2u * hl * tf_bits;
          const uint8_t* a0 = qw_smem + blk + 16u * doc_bits + ((bp0 >> 5) << 4);
          const uint4 A0 = *(const uint4*)a0, B0 = *(const uint4*)(a0 + 16);
          const uint32_t sh0 = bp0 & 31u;
          const uint32_t mask = __funnelshift_lc(0xFFFFFFFFu, 0u, tf_bits);
          const uint32_t x0 = __funnelshift_r(A0.x, B0.x, sh0), x1 = __funnelshift_r(A0.y, B0.y, sh0);
          const uint32_t x2 = __funnelshift_r(A0.z, B0.z, sh0), x3 = __funnelshift_r(A0.w, B0.w, sh0);
          f[0] = x0 & mask; f[1] = x1 & mask; f[2] = x2 & mask; f[3] = x3 & mask;
          f[4] = (x0 >> tf_bits) & mask; f[5] = (x1 >> tf_bits) & mask; f[6] = (x2 >> tf_bits) & mask; f[7] = (x3 >> tf_bits) & mask;
        } else if (tf_bits) {
          const uint32_t bp0 = 2u * hl * tf_bits, bp1 = bp0 + tf_bits;
          const uint8_t* a0 = qw_smem + blk + 16u * doc_bits + ((bp0 >> 5) << 4);
          const uint8_t* a1 = qw_smem + blk + 16u * doc_bits + ((bp1 >> 5) << 4);
          const uint4 A0 = *(const uint4*)a0, B0 = *(const uint4*)(a0 + 16);
          const uint4 A1 = *(const uint4*)a1, B1 = *(const uint4*)(a1 + 16);
          const uint32_t sh0 = bp0 & 31u, sh1 = bp1 & 31u;
          const uint32_t mask = __funnelshift_lc(0xFFFFFFFFu, 0u, tf_bits);
          f[0] = __funnelshift_r(A0.x, B0.x, sh0) & mask;
          f[1] = __funnelshift_r(A0.y, B0.y, sh0) & mask;
          f[2] = __funnelshift_r(A0.z, B0.z, sh0) & mask;
          f[3] = __funnelshift_r(A0.w, B0.w, sh0) & mask;
          f[4] = __funnelshift_r(A1.x, B1.x, sh1) & mask;
          f[5] = __funnelshift_r(A1.y, B1.y, sh1) & mask;
          f[6] = __funnelshift_r(A1.z, B1.z, sh1) & mask;
          f[7] = __funnelshift_r(A1.w, B1.w, sh1) & mask;
        }
        // ---- BM25: weight * (tf / (tf + norm[fieldnorm id])) from the tf-factor table ----------------
        uint2 fnw = make_uint2(0x01010101u, 0x01010101u);  // no fieldnorms: constant fieldnorm id 1
        if (tt.y & IF_HAS_FN) fnw = *(const uint2*)(qw_smem + blk + 16u * (doc_bits + tf_bits) + 8u * hl);
        float c[8];
        if (__all_sync(QW_FULL, tf_bits <= 4)) {
          // tf < 16: index = tf * 256 + fieldnorm id, one byte-permute per posting
          c[0] = __fmul_rn(weight, __ldg(tab + 256 + __byte_perm(f[0], fnw.x, 0x2104)));
          c[1] = __fmul_rn(weight, __ldg(tab + 256 + __byte_perm(f[1], fnw.x, 0x2105)));
          c[2] = __fmul_rn(weight, __ldg(tab + 256 + __byte_perm(f[2], fnw.x, 0x2106)));
          c[3] = __fmul_rn(weight, __ldg(tab + 256 + __byte_perm(f[3], fnw.x, 0x2107)));
          c[4] = __fmul_rn(weight, __ldg(tab + 256 + __byte_perm(f[4], fnw.y, 0x2104)));
          c[5] = __fmul_rn(weight, __ldg(tab + 256 + __byte_perm(f[5], fnw.y, 0x2105)));
          c[6] = __fmul_rn(weight, __ldg(tab + 256 + __byte_perm(f[6], fnw.y, 0x2106)));
          c[7] = __fmul_rn(weight, __ldg(tab + 256 + __byte_perm(f[7], fnw.y, 0x2107)));
        } else {
#pragma unroll
          for (int j = 0; j < 8; j++) {
            const uint32_t fn = ((j < 4 ? fnw.x : fnw.y) >> (8 * (j & 3))) & 0xFFu;
            c[j] = __fmul_rn(weight, tf_factor(tab, f[j], fn));
          }
        }
        // ---- ordered accumulate: everything of the earlier clauses must be in -------------------------
        const uint32_t count = rec.z >> 16;
        const uint32_t nvalid = !on ? 0u : (count > hl * 8u ? count - hl * 8u : 0u);  // postings of this lane that exist
        const bool all_interior = __all_sync(QW_FULL, on && (rec.w & 256u));
        auto apply = [&]() {
          if (all_interior) {
            // both blocks: all 128 postings exist and lie inside the window
            float o[8];
#pragma unroll
            for (int j = 0; j < 8; j++) o[j] = score[r[j]];
#pragma unroll
            for (int j = 0; j < 8; j++) score[r[j]] = __fadd_rn(o[j], c[j]);
          } else {
            float o[8];
            bool in[8];
#pragma unroll
            for (int j = 0; j < 8; j++) {
              in[j] = (uint32_t)j < nvalid && r[j] < wlen;  // r = doc - ws (unsigned wrap before the window)
              o[j] = 0.f;
              if (in[j]) o[j] = score[r[j]];
            }
#pragma unroll
            for (int j = 0; j < 8; j++) if (in[j]) score[r[j]] = __fadd_rn(o[j], c[j]);
          }
        };
        wait_below(st_lo);
        if (st_hi == st_lo || st_hi == 0u) apply();  // (lanes of an absent upper block have nvalid == 0)
        else {
          // the two blocks belong to different clauses: lower clause first
          if (half == 0) apply();
          pass_to(st_hi);  // (syncs the warp first: the lower block's stores are done)
          wait_below(st_hi);
          if (half == 1) apply();
        }
      }
      // this warp is done reading the slot (SAMPLE_COLLECT: the last slot of the block's first window -- wbase 1 -- is
      // held: its payload takes the sample's histogram, and the producer stages ahead into the other slot meanwhile)
      __syncwarp();
      const bool hold = MODE == MODE_SAMPLE_COLLECT && wbase == 1u && (flags & QU_F_LAST);
      if (lane == 0 && !hold) mbar_arrive(bar_empty(slot));
      if (!(flags & QU_F_LAST)) {
        pass_to(wbase + t_last);  // the slot's last clause may continue in the next slot
        continue;
      }
      const uint32_t end_stage = wbase + n_terms;
      pass_to(end_stage);
      // one group of four docs: scores (0 = no match); the accumulator is cleared on the way
      float4* sc4 = reinterpret_cast<float4*>(score);
      auto quad = [&](uint32_t q, float (&vv)[4]) {
        const float4 v = sc4[q];
        sc4[q] = make_float4(0.f, 0.f, 0.f, 0.f);
        vv[0] = v.x; vv[1] = v.y; vv[2] = v.z; vv[3] = v.w;
      };
      (void)quad;
      if (MODE == MODE_COLLECT) {
        // ---- sweep: count matches (score > 0), test against the threshold, clear ----------------------
        next_base = end_stage + 1;
        collect_sweep(ws, split, hdr_f, end_stage);
      } else if (MODE == MODE_SAMPLE_COLLECT) {
        next_base = end_stage + 1;
        if (hold) {
          // ---- the block's first window is its share of the threshold sample ---------------------------------
          wait_below(end_stage);  // every contribution is in, and no warp reads the slot any more
          auto consumers_sync = [&]() { asm volatile("bar.sync 1, %0;" ::"n"(QU_NCT) : "memory"); };
          uint32_t* shist = (uint32_t*)(qw_smem + sl + p.sm.payload);
          for (uint32_t i = tid; i < QW_HIST_BINS; i += QU_NCT) shist[i] = 0;
          consumers_sync();
          const DSplitPlan& P = p.plans[split];
          const float scale = P.key.score_scale;
          for (uint32_t q = tid; q < (W >> 2); q += QU_NCT) {
            const float4 v = sc4[q];  // (kept: the window is swept below, against the picked threshold)
            const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int j = 0; j < 4; j++) if (vv[j] > 0.0f) atomicAdd(&shist[score_digit(vv[j], scale)], 1u);
          }
          consumers_sync();
          flush_hist(P, shist, 1, false, tid, QU_NCT);
          consumers_sync();
          if (tid == 0 && !grid_barrier(p.sync, gridDim.x)) *p.err = 1;
          consumers_sync();
          // every block reads the same complete histograms: the same thresholds everywhere. The chunk touches the
          // split of its first window and at most one more (qw_fused_sample_plan: every split holds a first window).
          uint32_t split_b = split;
          while (__ldg(p.wl.first_work + split_b + 1) < w_end) split_b++;
          for (uint32_t k = 0; k < (split_b != split ? 2u : 1u); k++) {
            const uint32_t s = k ? split_b : split;
            const DSplitPlan& Ps = p.plans[s];
            if (Ps.max_hits == 0) { if (tid == 0) s_thr[k] = DThresh{}; }
            else if (warp < 256 / 32)  // (s_part, s_sel in the histogram's place, dead now)
              pick_digit<256>(Ps, s_thr[k], (const uint32_t*)Ps.out_hist, 0, 1, __ldg(p.sample_stride + s), tid, 2, shist, shist + 8);
          }
          consumers_sync();
          if (tid < 2) {
            const uint32_t s = tid ? split_b : split;
            s_thr_split[tid] = s;
            s_thr_lo[tid] = thresh_s_lo(s_thr[tid], p.plans[s].key.score_scale);
            // for the host and later passes: written by the lowest block whose chunk touches the split
            if (tid ? split_b != split : w_begin == __ldg(p.wl.first_work + split)) p.thresh[s] = s_thr[tid];
          }
          consumers_sync();
          if (lane == 0) mbar_arrive(bar_empty(slot));  // the held slot goes back to the producer
        }
        collect_sweep(ws, split, s_thr_lo[split == s_thr_split[0] ? 0 : 1], end_stage);
      } else {
        // level-0 digit histogram of the sampled windows: digit = [1 | lin:10] (score_lin)
        wait_below(end_stage);  // every contribution of the window is in
        const float scale = hdr_f;
        for (uint32_t q = tid; q < (W >> 2); q += QU_NCT) {
          float vv[4];
          quad(q, vv);
#pragma unroll
          for (int j = 0; j < 4; j++) if (vv[j] > 0.0f) atomicAdd(&hist[score_digit(vv[j], scale)], 1u);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_chain(end_stage));
        my_stage = end_stage + 1;
        wait_below(end_stage + 1);  // every warp has swept: the window's histogram is complete
        flush_hist(p.plans[split], hist, 1, true, tid, QU_NCT);
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_chain(end_stage + 1));
        my_stage = end_stage + 2;
        next_base = end_stage + 2;
      }
    }
    flush_hits();
  }
}

}  // namespace qwk
