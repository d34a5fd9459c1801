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

// one posting block of a phrase term by a warp (posting.cuh): docs (absolute), tfs (0 for padding postings, which own
// no positions) and their exclusive prefix over the block in lane-major order = each posting's first position index
// relative to the block's; returns the block's posting count
__device__ __forceinline__ uint32_t phrase_block(const uint8_t* blk, uint32_t lane, uint32_t (&doc)[4], uint32_t (&tf)[4], uint32_t (&pre)[4]) {
  const BlkHdr h = blk_header<LdgLoad>(blk);
  blk_docs<LdgLoad>(blk, h, 0, lane, doc);
  blk_tfs<LdgLoad>(blk, h, lane, tf);
#pragma unroll
  for (int j = 0; j < 4; j++) if (lane * 4 + j >= h.count) tf[j] = 0;
  const uint32_t s = tf[0] + tf[1] + tf[2] + tf[3];
  uint32_t incl = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t n = __shfl_up_sync(0xFFFFFFFFu, incl, o);
    if ((int)lane >= o) incl += n;
  }
  pre[0] = incl - s; pre[1] = pre[0] + tf[0]; pre[2] = pre[1] + tf[1]; pre[3] = pre[2] + tf[2];
  return h.count;
}

// Looks the live candidates of one driver block (bit j of `live`: doc cdoc[j]; the block spans [doc_first, doc_last])
// up in term T. The candidates form one contiguous doc range, so the blocks of T that can hold them are a short run
// [r_lo, r_hi]: two warp-cooperative searches find it (a handful of load rounds), and each candidate then searches
// inside it (one or two steps for terms of comparable density) instead of the whole skip list. The warp decodes each
// NEEDED block once, lowest first, into its shared arrays bdoc / bpre / btf (128 words each), and every candidate calls
// found(j, first position index, tf) or missing(j).
template <class Found, class Missing>
__device__ __forceinline__ void phrase_probe(const uint8_t* base, const DPhraseTerm& T, uint32_t doc_first, uint32_t doc_last,
                                             const uint32_t (&cdoc)[4], uint32_t live, uint32_t* bdoc, uint32_t* bpre,
                                             uint32_t* btf, uint32_t lane, Found&& found, Missing&& missing) {
  const QwSkip* sk = (const QwSkip*)(base + T.skip_off);
  const uint32_t* pidx = (const uint32_t*)(base + T.pidx_off);
  const uint32_t r_lo = first_block_ge(sk, T.nblk, doc_first, lane);
  const uint32_t r_hi = r_lo < T.nblk ? r_lo + first_block_ge(sk + r_lo, T.nblk - r_lo, doc_last, lane) : T.nblk;  // first block that reaches doc_last
  uint32_t need[4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    need[j] = QP_NONE;
    if ((live >> j) & 1u) {
      // first block whose last_doc >= doc
      uint32_t lo = r_lo, hi = min(r_hi + 1, T.nblk);
      while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (__ldg(&sk[mid].last_doc) < cdoc[j]) lo = mid + 1; else hi = mid;
      }
      if (lo < T.nblk) need[j] = lo; else missing(j);
    }
  }
  for (;;) {
    uint32_t cur = min(min(need[0], need[1]), min(need[2], need[3]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cur = min(cur, __shfl_xor_sync(0xFFFFFFFFu, cur, o));
    if (cur == QP_NONE) break;
    // the warp decodes block `cur` of term T into shared memory
    uint32_t d[4], f[4], pre[4];
    const uint32_t cnt = phrase_block(base + T.data_off + __ldg(&sk[cur].byte_off), lane, d, f, pre);
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
      if (lo < cnt && bdoc[lo] == cdoc[j]) found(j, first + bpre[lo], btf[lo]);
      else missing(j);
    }
  }
}

// A driver block's result as an uncompressed posting block: candidate j with phrase_count n[j] > 0 is {doc, weight *
// tf-factor(n[j], fieldnorm)} (Bm25Weight::score with tf = phrase_count; val 0 when the phrase is unscored); the others
// are {QP_NONE, 0}
__device__ __forceinline__ void phrase_out(const DPhrase& ph, const uint8_t* base, uint32_t b, uint32_t lane, const uint32_t (&cdoc)[4],
                                           const uint32_t (&n)[4]) {
  uint32_t odoc[4];
  float oval[4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    odoc[j] = n[j] ? cdoc[j] : QP_NONE;
    oval[j] = 0.f;
    if (n[j] && ph.scored) {
      const uint32_t fn = ph.fn_off != ~0ull ? (uint32_t)__ldg(base + ph.fn_off + cdoc[j]) : 1u;
      oval[j] = __fmul_rn(ph.weight, tf_factor((const float*)ph.tab, n[j], fn));
    }
  }
  VBlk* out = (VBlk*)ph.out + b;
  *reinterpret_cast<uint4*>(&out->doc[lane * 4]) = make_uint4(odoc[0], odoc[1], odoc[2], odoc[3]);
  *reinterpret_cast<float4*>(&out->val[lane * 4]) = make_float4(oval[0], oval[1], oval[2], oval[3]);
}

// shared memory per warp: 3 + 2 * max_terms arrays of 128 words (max_terms = the longest phrase of the batch), so that
// short phrases — the usual case — leave room for three times as many warps per SM as a layout sized for 8 terms
#define QP_SMEM_WORDS(max_terms) ((3u + 2u * (max_terms)) * QW_BLOCK_LEN)
// kPrefix: the batch holds at least one phrase prefix (n_exp > 0); its plain phrases take the same path as in
// k_phrase<false>. k_phrase<false> asks for 10 blocks per SM (at most 48 registers): left to itself the compiler
// takes 56 registers and no spills, and a batch of many short phrases then runs about 5% slower on an H100.
template <bool kPrefix>
__global__ void __launch_bounds__(QP_WARPS * 32, kPrefix ? 0 : 10) k_phrase(const DPhrase* phrases, uint32_t n_phrases, uint32_t total_blocks, uint32_t max_terms) {
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
    count = phrase_block(base + D.data_off + __ldg(&sk[b].byte_off), lane, cdoc, ctf, cpre);
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
    const uint32_t doc_first = __shfl_sync(0xFFFFFFFFu, cdoc[0], 0);
    const uint32_t doc_last = __ldg(&((const QwSkip*)(base + D.skip_off))[b].last_doc);
    phrase_probe(base, ph.t[t], doc_first, doc_last, cdoc, alive, bdoc, bpre, btf, lane,
                 [&](uint32_t j, uint32_t pos, uint32_t tf) { S_POS(t, lane * 4 + j) = pos; S_TF(t, lane * 4 + j) = tf; },
                 [&](uint32_t j) { alive &= ~(1u << j); });
  }

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
        phrase_probe(base, T, doc_first, doc_last, cdoc, open, bdoc, bpre, btf, lane,
                     [&](uint32_t j, uint32_t pos, uint32_t ne) {
                       const uint32_t c = lane * 4 + j;
                       const uint32_t* pe = (const uint32_t*)(base + T.pos_off) + pos;
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
                     },
                     [](uint32_t) {});
      }
      uint32_t odoc[4];
#pragma unroll
      for (int j = 0; j < 4; j++) odoc[j] = (matched >> j) & 1u ? cdoc[j] : QP_NONE;
      VBlk* out = (VBlk*)ph.out + b;
      *reinterpret_cast<uint4*>(&out->doc[lane * 4]) = make_uint4(odoc[0], odoc[1], odoc[2], odoc[3]);
      *reinterpret_cast<float4*>(&out->val[lane * 4]) = make_float4(0.f, 0.f, 0.f, 0.f);
      return;
    }
  }

  // ---- 3. positions: base positions at which every term lines up -----------------------------------------------
  const uint32_t off_d = D.offset;
  uint32_t matches[4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    matches[j] = 0;
    if (!((alive >> j) & 1u)) continue;
    const uint32_t c = lane * 4 + j;
    const uint32_t* pd = (const uint32_t*)(base + D.pos_off) + S_POS(ph.driver, c);
    const uint32_t nd = ctf[j];
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
      matches[j] += all ? 1u : 0u;
    }
  }
  phrase_out(ph, base, b, lane, cdoc, matches);
}

// ---- phrases of more than QW_MAX_PHRASE_TERMS terms (k_phrase_long) ------------------------------------------------
// k_phrase keeps every term's {first position index, tf} of all 128 candidates in shared memory, which grows with the
// phrase. The long pre-pass keeps no per-term state: its terms (ph.exp, the driver first, then by ascending doc_freq)
// are taken once each, and every present candidate at once narrows its surviving base positions to those where the
// term lines up. The survivors are a 32-bit mask over one round of 32 driver positions; a candidate whose driver tf
// exceeds 32 takes the term loop again for each further round of 32. A candidate dies when it lacks a term or its
// mask empties, and a round ends as soon as no candidate of the warp holds a survivor, so a mismatch at an early term
// costs that term only. Shared memory per warp: the decoded block of the term being probed, whatever the length.

// the bits i of `mask` whose base pd[i] - off_d has a position base + off_t among the sorted pt[0, nt)
__device__ __forceinline__ uint32_t phrase_narrow(const uint32_t* pd, uint32_t mask, uint32_t off_d, const uint32_t* pt,
                                                  uint32_t nt, uint32_t off_t) {
  uint32_t keep = 0, from = 0;
  while (mask) {
    const uint32_t i = __ffs(mask) - 1;
    mask &= mask - 1;
    const uint32_t p = __ldg(pd + i);
    if (p < off_d) continue;  // the phrase would start before position 0
    const uint32_t want = p - off_d + off_t;
    uint32_t lo = from, hi = nt;  // the wanted positions ascend with i: search past the previous hit only
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      if (__ldg(pt + mid) < want) lo = mid + 1; else hi = mid;
    }
    if (lo == nt) break;
    from = lo;
    if (__ldg(pt + lo) == want) keep |= 1u << i;
  }
  return keep;
}

__global__ void __launch_bounds__(QP_WARPS * 32) k_phrase_long(const DPhrase* phrases, uint32_t n_phrases, uint32_t total_blocks) {
  __shared__ __align__(16) uint32_t ql_smem[QP_WARPS][3 * QW_BLOCK_LEN];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t* bdoc = ql_smem[warp]; uint32_t* bpre = bdoc + QW_BLOCK_LEN; uint32_t* btf = bdoc + 2 * QW_BLOCK_LEN;
  const uint32_t work = blockIdx.x * QP_WARPS + warp;
  if (work >= total_blocks) return;
  uint32_t pi = 0;
  while (pi + 1 < n_phrases && phrases[pi + 1].first_work <= work) pi++;
  const DPhrase& ph = phrases[pi];
  const uint32_t b = work - ph.first_work;
  const uint8_t* base = (const uint8_t*)ph.data_base;
  const DPhraseTerm* terms = (const DPhraseTerm*)ph.exp;
  const DPhraseTerm& D = terms[0];

  // ---- 1. driver block ------------------------------------------------------------------------------------
  const QwSkip* dsk = (const QwSkip*)(base + D.skip_off);
  uint32_t cdoc[4], ctf[4], cpre[4];
  const uint32_t count = phrase_block(base + D.data_off + __ldg(&dsk[b].byte_off), lane, cdoc, ctf, cpre);
  const uint32_t* dpos = (const uint32_t*)(base + D.pos_off) + __ldg((const uint32_t*)(base + D.pidx_off) + b);
  const uint32_t off_d = D.offset;
  const uint32_t doc_first = __shfl_sync(0xFFFFFFFFu, cdoc[0], 0);
  const uint32_t doc_last = __ldg(&dsk[b].last_doc);
  uint32_t present = 0;  // bit j: candidate j holds every term looked up so far
#pragma unroll
  for (int j = 0; j < 4; j++) if (lane * 4 + j < count) present |= 1u << j;
  uint32_t matches[4] = {0, 0, 0, 0};

  // ---- 2. rounds of 32 driver positions, each narrowed by the other terms in order ------------------------------
  for (uint32_t r0 = 0;; r0 += 32) {
    uint32_t mask[4], live = 0;  // live bit j: candidate j still has a survivor in this round
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const uint32_t left = ((present >> j) & 1u) && ctf[j] > r0 ? ctf[j] - r0 : 0u;
      mask[j] = left >= 32 ? 0xFFFFFFFFu : (1u << left) - 1u;
      if (left) live |= 1u << j;
    }
    if (!__ballot_sync(0xFFFFFFFFu, live != 0)) break;
    for (uint32_t t = 1; t < ph.n_terms; t++) {
      const DPhraseTerm& T = terms[t];
      const uint32_t* tpos = (const uint32_t*)(base + T.pos_off);
      phrase_probe(base, T, doc_first, doc_last, cdoc, live, bdoc, bpre, btf, lane,
                   [&](uint32_t j, uint32_t pos, uint32_t tf) {
                     mask[j] = phrase_narrow(dpos + cpre[j] + r0, mask[j], off_d, tpos + pos, tf, T.offset);
                     if (!mask[j]) live &= ~(1u << j);
                   },
                   [&](uint32_t j) { present &= ~(1u << j); live &= ~(1u << j); mask[j] = 0; });
      if (!__ballot_sync(0xFFFFFFFFu, live != 0)) break;  // no survivor left in the warp: the later terms are moot
    }
#pragma unroll
    for (int j = 0; j < 4; j++) matches[j] += __popc(mask[j]);
  }

  // ---- 3. output: k_phrase's scoring of phrase_count = matches ------------------------------------------------
  phrase_out(ph, base, b, lane, cdoc, matches);
}

}  // namespace qwk
