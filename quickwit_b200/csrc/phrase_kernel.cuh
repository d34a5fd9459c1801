// phrase_kernel.cuh — tantivy PhraseQuery (slop 0) as a pre-pass that turns a phrase into a posting list.
//
// Replaces PhraseScorer (tantivy phrase_scorer.rs: intersection of the terms' docsets, then of their position
// lists shifted by the terms' offsets) + PhraseWeight's Bm25Weight::for_terms behind `searcher.search`
// (quickwit-search/src/leaf.rs:637) for QueryAst full_text mode `phrase`
// (quickwit-query/src/query_ast/full_text_query.rs:140-156). SURVEY.md 8f-1.
//
// The rarest term of the phrase drives: one warp per 128-posting block of the driver term.
//   1. the warp decodes the driver block (doc ids, tfs -> first position index of every posting);
//   2. per other term: every lane finds, for its four candidate docs, the posting block that can hold the doc
//      (binary search of the skip list); the warp then decodes each NEEDED block once, lowest first, into shared
//      memory and the lanes look their candidates up in it (doc -> tf and first position index);
//   3. candidates present in every term: the positions of the driver posting are matched against the other
//      terms' position ranges (binary search), phrase_count = number of base positions where all terms line up;
//   4. the block's result is written as an uncompressed posting block {doc or NONE, f32 contribution}[128]
//      (contribution = weight * tf-factor(phrase_count, fieldnorm), the same table / divide as a term's BM25).
// The window kernel then consumes the phrase like a term whose blocks are already decoded (OP_PHRASE,
// kernels.cuh::fold_vblock), finding the blocks of a window through the driver term's skip list.
//
// A phrase prefix (tantivy PhrasePrefixQuery, QW_NODE_PHRASE_PREFIX) is the same pre-pass over its exact terms, the
// rarest of them driving, whose last slot is a SET of terms (the prefix's expansions). Step 3 is replaced by a suffix
// stage (2b): per expansion, in order, the candidates still alive and not yet matched are looked up in the
// expansion's blocks like in step 2, and every position q >= offset_last of a present candidate tests the base
// b = q - offset_last against every exact term's positions. The loop ends once every alive candidate of the warp has
// matched. The output is unscored (val = 0). Only the k_phrase<true> instantiation carries the stage, so batches
// without a phrase prefix run the plain kernel unchanged.
#pragma once
#include "kernels.cuh"

namespace qwk {

#define QP_WARPS 4
#define QP_NONE 0xFFFFFFFFu

// block-wide unpack of one posting block by a warp: docs (absolute) and tfs of the lane's 4 postings
__device__ __forceinline__ void phrase_decode(const uint8_t* blk, uint32_t lane, uint32_t (&doc)[4], uint32_t (&tf)[4], uint32_t& count) {
  const uint4 h = __ldg(reinterpret_cast<const uint4*>(blk));  // QwSkip: last_doc, prev_last_doc, byte_off, bits/count
  const uint32_t prev = h.y, doc_bits = h.w & 0xFF, tf_bits = (h.w >> 8) & 0xFF;
  count = h.w >> 16;
  const uint4* dp = reinterpret_cast<const uint4*>(blk + 16);
  uint32_t v[4] = {0, 0, 0, 0};
  if (doc_bits) {
    const uint32_t bitpos = lane * doc_bits, wi = bitpos >> 5, sh = bitpos & 31;
    const uint4 A = __ldg(dp + wi);
    const uint4 B = (sh + doc_bits > 32) ? __ldg(dp + wi + 1) : make_uint4(0, 0, 0, 0);
    const uint32_t mask = 0xFFFFFFFFu >> (32 - doc_bits);
    v[0] = __funnelshift_r(A.x, B.x, sh) & mask; v[1] = __funnelshift_r(A.y, B.y, sh) & mask;
    v[2] = __funnelshift_r(A.z, B.z, sh) & mask; v[3] = __funnelshift_r(A.w, B.w, sh) & mask;
  }
  const uint32_t d0 = v[0] + 1, d1 = d0 + v[1] + 1, d2 = d1 + v[2] + 1, d3 = d2 + v[3] + 1;
  uint32_t incl = d3;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t n = __shfl_up_sync(0xFFFFFFFFu, incl, o);
    if ((int)lane >= o) incl += n;
  }
  const uint32_t basev = prev + (incl - d3);  // mod 2^32
  doc[0] = basev + d0; doc[1] = basev + d1; doc[2] = basev + d2; doc[3] = basev + d3;
  tf[0] = tf[1] = tf[2] = tf[3] = 1;
  if (tf_bits) {
    const uint4* tp = dp + doc_bits;
    const uint32_t bitpos = lane * tf_bits, wi = bitpos >> 5, sh = bitpos & 31;
    const uint4 A = __ldg(tp + wi);
    const uint4 B = (sh + tf_bits > 32) ? __ldg(tp + wi + 1) : make_uint4(0, 0, 0, 0);
    const uint32_t mask = 0xFFFFFFFFu >> (32 - tf_bits);
    tf[0] = __funnelshift_r(A.x, B.x, sh) & mask; tf[1] = __funnelshift_r(A.y, B.y, sh) & mask;
    tf[2] = __funnelshift_r(A.z, B.z, sh) & mask; tf[3] = __funnelshift_r(A.w, B.w, sh) & mask;
  }
#pragma unroll
  for (int j = 0; j < 4; j++) if (lane * 4 + j >= count) tf[j] = 0;  // padding postings own no positions
}

// exclusive prefix of the lane's 4 values over the whole block (lane-major order)
__device__ __forceinline__ void block_excl_prefix(const uint32_t (&x)[4], uint32_t lane, uint32_t (&pre)[4]) {
  const uint32_t s = x[0] + x[1] + x[2] + x[3];
  uint32_t incl = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t n = __shfl_up_sync(0xFFFFFFFFu, incl, o);
    if ((int)lane >= o) incl += n;
  }
  pre[0] = incl - s; pre[1] = pre[0] + x[0]; pre[2] = pre[1] + x[1]; pre[3] = pre[2] + x[2];
}

// first index in [0, n) whose skip entry has last_doc >= doc (n if none): warp-cooperative 32-ary search, one round
// of coalesced loads per factor 32
__device__ __forceinline__ uint32_t phrase_first_block(const QwSkip* sk, uint32_t n, uint32_t doc, uint32_t lane) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t step = (hi - lo + 31) / 32, idx = lo + lane * step;
    const bool before = idx < hi && __ldg(&sk[idx].last_doc) < doc;  // true for a prefix of the probes
    const uint32_t c = (uint32_t)__popc(__ballot_sync(0xFFFFFFFFu, before));
    if (c == 0) { hi = lo; break; }
    hi = min(hi, lo + c * step);
    lo = lo + (c - 1) * step + 1;
  }
  return lo;
}

// shared memory per warp: 3 + 2 * max_terms arrays of 128 words (max_terms = the longest phrase of the batch), so that
// short phrases — the usual case — leave room for three times as many warps per SM as a layout sized for 8 terms
#define QP_SMEM_WORDS(max_terms) ((3u + 2u * (max_terms)) * QW_BLOCK_LEN)
// kPrefix: the batch holds at least one phrase prefix (n_exp > 0); its plain phrases take the same path as in
// k_phrase<false>
template <bool kPrefix>
__global__ void __launch_bounds__(QP_WARPS * 32) k_phrase(const DPhrase* phrases, uint32_t n_phrases, uint32_t total_blocks, uint32_t max_terms) {
  // per warp: the decoded block of the term being probed + every term's {first position index, tf} per candidate
  extern __shared__ __align__(16) uint8_t qp_smem[];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t* wsm = (uint32_t*)qp_smem + (size_t)warp * QP_SMEM_WORDS(max_terms);
  uint32_t* bdoc = wsm; uint32_t* bpre = wsm + QW_BLOCK_LEN; uint32_t* btf = wsm + 2 * QW_BLOCK_LEN;
  uint32_t* s_pos_w = wsm + 3 * QW_BLOCK_LEN;                              // [max_terms][128]
  uint32_t* s_tf_w = s_pos_w + (size_t)max_terms * QW_BLOCK_LEN;           // [max_terms][128]
#define S_POS(t, c) s_pos_w[(t) * QW_BLOCK_LEN + (c)]
#define S_TF(t, c) s_tf_w[(t) * QW_BLOCK_LEN + (c)]
  const uint32_t work = blockIdx.x * QP_WARPS + warp;
  if (work >= total_blocks) return;
  // which phrase, which driver block
  uint32_t pi = 0;
  while (pi + 1 < n_phrases && phrases[pi + 1].first_work <= work) pi++;
  const DPhrase& ph = phrases[pi];
  const uint32_t b = work - ph.first_work;
  const uint8_t* base = (const uint8_t*)ph.data_base;
  const DPhraseTerm& D = ph.t[ph.driver];

  // ---- 1. driver block ------------------------------------------------------------------------------------
  uint32_t cdoc[4], ctf[4], cpre[4], count;
  {
    const QwSkip* sk = (const QwSkip*)(base + D.skip_off);
    phrase_decode(base + D.data_off + __ldg(&sk[b].byte_off), lane, cdoc, ctf, count);
    block_excl_prefix(ctf, lane, cpre);
    const uint32_t first = __ldg((const uint32_t*)(base + D.pidx_off) + b);
#pragma unroll
    for (int j = 0; j < 4; j++) {
      S_POS(ph.driver, lane * 4 + j) = first + cpre[j];
      S_TF(ph.driver, lane * 4 + j) = ctf[j];
    }
  }
  uint32_t alive = 0;  // bit j: candidate j of this lane is still in every term seen so far
#pragma unroll
  for (int j = 0; j < 4; j++) if (lane * 4 + j < count) alive |= 1u << j;

  // ---- 2. the other terms ------------------------------------------------------------------------------------
  for (uint32_t t = 0; t < ph.n_terms; t++) {
    if (t == ph.driver) continue;
    const DPhraseTerm& T = ph.t[t];
    const QwSkip* sk = (const QwSkip*)(base + T.skip_off);
    const uint32_t* pidx = (const uint32_t*)(base + T.pidx_off);
    // The candidates are the postings of ONE driver block, i.e. a contiguous doc range: the blocks of term t that can
    // hold them form a short run [r_lo, r_hi]. Two warp-cooperative searches find the run (a handful of load rounds);
    // each candidate then searches inside it (one or two steps for terms of comparable density) instead of the whole
    // skip list (14 dependent loads for 10 K blocks, four times per lane).
    const uint32_t doc_first = __shfl_sync(0xFFFFFFFFu, cdoc[0], 0);
    const uint32_t doc_last = __ldg(&((const QwSkip*)(base + D.skip_off))[b].last_doc);
    const uint32_t r_lo = phrase_first_block(sk, T.nblk, doc_first, lane);
    const uint32_t r_hi = r_lo < T.nblk ? r_lo + phrase_first_block(sk + r_lo, T.nblk - r_lo, doc_last, lane) : T.nblk;  // first block that reaches doc_last
    uint32_t need[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      need[j] = QP_NONE;
      if ((alive >> j) & 1u) {
        // first block whose last_doc >= doc
        uint32_t lo = r_lo, hi = min(r_hi + 1, T.nblk);
        while (lo < hi) {
          const uint32_t mid = (lo + hi) >> 1;
          if (__ldg(&sk[mid].last_doc) < cdoc[j]) lo = mid + 1; else hi = mid;
        }
        if (lo < T.nblk) need[j] = lo; else alive &= ~(1u << j);
      }
    }
    for (;;) {
      uint32_t cur = min(min(need[0], need[1]), min(need[2], need[3]));
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) cur = min(cur, __shfl_xor_sync(0xFFFFFFFFu, cur, o));
      if (cur == QP_NONE) break;
      // the warp decodes block `cur` of term t into shared memory
      uint32_t d[4], f[4], pre[4], cnt;
      phrase_decode(base + T.data_off + __ldg(&sk[cur].byte_off), lane, d, f, cnt);
      block_excl_prefix(f, lane, pre);
      __syncwarp();
#pragma unroll
      for (int j = 0; j < 4; j++) {
        bdoc[lane * 4 + j] = lane * 4 + j < cnt ? d[j] : QP_NONE;  // (padding sorts last)
        bpre[lane * 4 + j] = pre[j];
        btf[lane * 4 + j] = f[j];
      }
      __syncwarp();
      const uint32_t first = __ldg(pidx + cur);
#pragma unroll
      for (int j = 0; j < 4; j++) {
        if (need[j] != cur) continue;
        need[j] = QP_NONE;
        uint32_t lo = 0, hi = cnt;
        while (lo < hi) {
          const uint32_t mid = (lo + hi) >> 1;
          if (bdoc[mid] < cdoc[j]) lo = mid + 1; else hi = mid;
        }
        if (lo < cnt && bdoc[lo] == cdoc[j]) {
          S_POS(t, lane * 4 + j) = first + bpre[lo];
          S_TF(t, lane * 4 + j) = btf[lo];
        } else alive &= ~(1u << j);
      }
    }
  }

  VBlk* out = (VBlk*)ph.out + b;
  if constexpr (kPrefix) {
    if (ph.n_exp) {
      // ---- 2b. phrase prefix: the expansions of the last slot ----------------------------------------------------
      const DPhraseTerm* X = (const DPhraseTerm*)ph.exp;
      const uint32_t doc_first = __shfl_sync(0xFFFFFFFFu, cdoc[0], 0);
      const uint32_t doc_last = __ldg(&((const QwSkip*)(base + D.skip_off))[b].last_doc);
      uint32_t matched = 0;  // bit j: candidate j holds the phrase with some expansion
      for (uint32_t e = 0; e < ph.n_exp; e++) {
        const uint32_t open = alive & ~matched;
        if (!__ballot_sync(0xFFFFFFFFu, open != 0)) break;  // every alive candidate of the warp has matched
        const DPhraseTerm& T = X[e];
        const QwSkip* sk = (const QwSkip*)(base + T.skip_off);
        const uint32_t* pidx = (const uint32_t*)(base + T.pidx_off);
        const uint32_t r_lo = phrase_first_block(sk, T.nblk, doc_first, lane);
        if (r_lo >= T.nblk) continue;  // every posting of the expansion lies before the driver block
        const uint32_t r_hi = r_lo + phrase_first_block(sk + r_lo, T.nblk - r_lo, doc_last, lane);
        uint32_t need[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
          need[j] = QP_NONE;
          if ((open >> j) & 1u) {
            uint32_t lo = r_lo, hi = min(r_hi + 1, T.nblk);
            while (lo < hi) {
              const uint32_t mid = (lo + hi) >> 1;
              if (__ldg(&sk[mid].last_doc) < cdoc[j]) lo = mid + 1; else hi = mid;
            }
            if (lo < T.nblk) need[j] = lo;
          }
        }
        for (;;) {
          uint32_t cur = min(min(need[0], need[1]), min(need[2], need[3]));
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) cur = min(cur, __shfl_xor_sync(0xFFFFFFFFu, cur, o));
          if (cur == QP_NONE) break;
          uint32_t d[4], f[4], pre[4], cnt;
          phrase_decode(base + T.data_off + __ldg(&sk[cur].byte_off), lane, d, f, cnt);
          block_excl_prefix(f, lane, pre);
          __syncwarp();
#pragma unroll
          for (int j = 0; j < 4; j++) {
            bdoc[lane * 4 + j] = lane * 4 + j < cnt ? d[j] : QP_NONE;
            bpre[lane * 4 + j] = pre[j];
            btf[lane * 4 + j] = f[j];
          }
          __syncwarp();
          const uint32_t first = __ldg(pidx + cur);
#pragma unroll
          for (int j = 0; j < 4; j++) {
            if (need[j] != cur) continue;
            need[j] = QP_NONE;
            uint32_t lo = 0, hi = cnt;
            while (lo < hi) {
              const uint32_t mid = (lo + hi) >> 1;
              if (bdoc[mid] < cdoc[j]) lo = mid + 1; else hi = mid;
            }
            if (lo >= cnt || bdoc[lo] != cdoc[j]) continue;
            const uint32_t c = lane * 4 + j;
            const uint32_t* pe = (const uint32_t*)(base + T.pos_off) + first + bpre[lo];
            const uint32_t ne = btf[lo];
            for (uint32_t i = 0; i < ne; i++) {
              const uint32_t q = __ldg(pe + i);
              if (q < T.offset) continue;  // the phrase would start before position 0
              const uint32_t start = q - T.offset;
              bool all = true;
              for (uint32_t t = 0; t < ph.n_terms && all; t++) {
                const uint32_t want = start + ph.t[t].offset;
                const uint32_t* pt = (const uint32_t*)(base + ph.t[t].pos_off) + S_POS(t, c);
                uint32_t plo = 0, phi = S_TF(t, c);
                while (plo < phi) {
                  const uint32_t mid = (plo + phi) >> 1;
                  if (__ldg(pt + mid) < want) plo = mid + 1; else phi = mid;
                }
                all = plo < S_TF(t, c) && __ldg(pt + plo) == want;
              }
              if (all) { matched |= 1u << j; break; }
            }
          }
        }
      }
      uint32_t odoc[4];
#pragma unroll
      for (int j = 0; j < 4; j++) odoc[j] = (matched >> j) & 1u ? cdoc[j] : QP_NONE;
      *reinterpret_cast<uint4*>(&out->doc[lane * 4]) = make_uint4(odoc[0], odoc[1], odoc[2], odoc[3]);
      *reinterpret_cast<float4*>(&out->val[lane * 4]) = make_float4(0.f, 0.f, 0.f, 0.f);
      return;
    }
  }

  // ---- 3. positions: base positions at which every term lines up -----------------------------------------------
  const uint32_t off_d = D.offset;
  uint32_t odoc[4];
  float oval[4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    odoc[j] = QP_NONE;
    oval[j] = 0.f;
    if (!((alive >> j) & 1u)) continue;
    const uint32_t c = lane * 4 + j;
    const uint32_t* pd = (const uint32_t*)(base + D.pos_off) + S_POS(ph.driver, c);
    const uint32_t nd = ctf[j];
    uint32_t matches = 0;
    for (uint32_t i = 0; i < nd; i++) {
      const uint32_t p = __ldg(pd + i);
      if (p < off_d) continue;  // the phrase would start before position 0
      const uint32_t start = p - off_d;
      bool all = true;
      for (uint32_t t = 0; t < ph.n_terms && all; t++) {
        if (t == ph.driver) continue;
        const uint32_t want = start + ph.t[t].offset;
        const uint32_t* pt = (const uint32_t*)(base + ph.t[t].pos_off) + S_POS(t, c);
        uint32_t lo = 0, hi = S_TF(t, c);
        while (lo < hi) {
          const uint32_t mid = (lo + hi) >> 1;
          if (__ldg(pt + mid) < want) lo = mid + 1; else hi = mid;
        }
        all = lo < S_TF(t, c) && __ldg(pt + lo) == want;
      }
      matches += all ? 1u : 0u;
    }
    if (matches) {
      odoc[j] = cdoc[j];
      if (ph.scored) {
        // Bm25Weight::score with tf = phrase_count: the same table / divide as a term posting
        const float* tab = (const float*)ph.tab;
        const uint32_t fn = ph.fn_off != ~0ull ? (uint32_t)__ldg(base + ph.fn_off + cdoc[j]) : 1u;
        float tfn;
        if (matches < QW_TFF_ROWS) tfn = __ldg(tab + 256 + matches * 256 + fn);
        else { const float tff = (float)matches; tfn = __fdiv_rn(tff, __fadd_rn(tff, __ldg(tab + fn))); }
        oval[j] = __fmul_rn(ph.weight, tfn);
      }
    }
  }
  *reinterpret_cast<uint4*>(&out->doc[lane * 4]) = make_uint4(odoc[0], odoc[1], odoc[2], odoc[3]);
  *reinterpret_cast<float4*>(&out->val[lane * 4]) = make_float4(oval[0], oval[1], oval[2], oval[3]);
}

}  // namespace qwk
