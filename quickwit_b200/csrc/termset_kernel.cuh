// termset_kernel.cuh — the doc-set pre-pass of QW_NODE_TERM_SET (regex expansions): the union of the postings of up to
// QW_MAX_SET_TERMS terms, as one bitmap of ceil(num_docs / 32) words per node, zeroed before the launch. The window
// program then ORs a window's words into the clause's target (OP_TERM_SET, kernels.cuh).
//
// One warp per 128-posting block, over the flat block list of every term-set term of the batch (grid-stride). A warp
// finds its term by a 32-ary search of the block prefix, decodes the block's doc ids (posting.cuh), and sets
// the doc bits with one atomicOr per distinct bitmap word: the block's postings are taken 32 at a time in doc order,
// __match_any_sync groups the lanes of one word (a contiguous run, since doc ids ascend), a segmented shuffle ORs the
// run into its first lane, and the run that ends a round is carried into the next round, which may continue the word.
#pragma once
#include "posting.cuh"

namespace qwk {

#define QS_WARPS 8

__global__ void __launch_bounds__(QS_WARPS * 32) k_term_set(const DTermSetTerm* terms, uint32_t n_terms, const DTermSetNode* nodes,
                                                            uint32_t total_blocks) {
  const uint32_t FULL = 0xFFFFFFFFu, NONE = 0xFFFFFFFFu;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t nwarps = gridDim.x * QS_WARPS;
  for (uint32_t b = blockIdx.x * QS_WARPS + (threadIdx.x >> 5); b < total_blocks; b += nwarps) {
    // the last term whose first block is <= b: terms[lo].first_block <= b < terms[hi].first_block
    uint32_t lo = 0, hi = n_terms;
    while (hi - lo > 1) {
      const uint32_t step = (hi - lo + 31) / 32, idx = lo + lane * step;
      const bool le = idx < hi && __ldg(&terms[idx].first_block) <= b;
      const uint32_t c = (uint32_t)__popc(__ballot_sync(FULL, le));  // >= 1: lane 0 probes lo
      lo += (c - 1) * step;
      hi = min(hi, lo + step);
    }
    const DTermSetTerm& T = terms[lo];
    const QwSkip* skips = (const QwSkip*)__ldg(&T.skip);
    const uint8_t* blk = (const uint8_t*)__ldg(&T.data) + __ldg(&skips[b - __ldg(&T.first_block)].byte_off);
    const BlkHdr h = blk_header<LdgLoad>(blk);
    uint32_t doc[4];
    blk_docs<LdgLoad>(blk, h, 0, lane, doc);
    uint32_t* bm = (uint32_t*)__ldg(&nodes[__ldg(&T.node)].bitmap);
    uint32_t carry = 0, carry_w = NONE;
#pragma unroll
    for (uint32_t r = 0; r < 4; r++) {
      // posting 32 r + lane (lane-major decode: lane l holds postings 4 l .. 4 l + 3)
      const uint32_t src = r * 8 + (lane >> 2), j = lane & 3;
      const uint32_t d0 = __shfl_sync(FULL, doc[0], src), d1 = __shfl_sync(FULL, doc[1], src);
      const uint32_t d2 = __shfl_sync(FULL, doc[2], src), d3 = __shfl_sync(FULL, doc[3], src);
      const uint32_t d = j == 0 ? d0 : j == 1 ? d1 : j == 2 ? d2 : d3;
      const bool valid = r * 32 + lane < h.count;
      const uint32_t w = valid ? d >> 5 : NONE;
      uint32_t v = valid ? 1u << (d & 31) : 0u;
      const uint32_t grp = __match_any_sync(FULL, w);
#pragma unroll
      for (uint32_t o = 1; o < 32; o <<= 1) {
        const uint32_t x = __shfl_down_sync(FULL, v, o), wx = __shfl_down_sync(FULL, w, o);
        if (lane + o < 32 && wx == w) v |= x;
      }
      const bool head = lane == (uint32_t)__ffs(grp) - 1;
      // the previous round's last run: continued by this round's first run, or written now
      if (head && w == carry_w) v |= carry;
      else if (lane == 0 && carry_w != NONE) atomicOr(bm + carry_w, carry);
      const uint32_t tail_w = __shfl_sync(FULL, w, 31);
      if (head && valid && !(w == tail_w && r < 3)) atomicOr(bm + w, v);
      const uint32_t tail_head = (uint32_t)__ffs(__shfl_sync(FULL, grp, 31)) - 1;
      carry = __shfl_sync(FULL, v, tail_head);
      carry_w = r < 3 ? tail_w : NONE;
    }
  }
}

}  // namespace qwk
