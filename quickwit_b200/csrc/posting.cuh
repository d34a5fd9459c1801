// posting.cuh — the one decoder of the image's posting blocks (qwgpu_format.h QwSkip) for the kernels that give a
// whole 128-posting block to one warp: k_window (fold_block), k_driver, k_phrase, k_phrase_long and k_term_set. Lane l
// holds postings 4 l .. 4 l + 3 (the 4-lane interleave). k_union decodes the same format its own way: half-warps,
// 8 postings per lane, from TMA-staged shared memory (union_kernel.cuh).
//
// A block is [16-byte header][doc deltas at doc_bits][tfs at tf_bits][128 fieldnorm ids if the field has them]. The
// steps stay separate because callers differ: fold_block rejects a block on its header before decoding anything, and
// only scored clauses of fields with frequencies read tfs.
#pragma once
#include <cuda_runtime.h>

#include "device_types.h"

namespace qwk {

// Load policies: `LdgLoad` reads global memory through the read-only data path; `PlainLoad` dereferences (staged
// blocks in shared memory, and k_window's direct mode).
struct LdgLoad {
  template <class T> __device__ __forceinline__ static T ld(const T* p) { return __ldg(p); }
};
struct PlainLoad {
  template <class T> __device__ __forceinline__ static T ld(const T* p) { return *p; }
};

struct BlkHdr {
  uint32_t last_doc, prev;  // prev: last doc of the previous block (QW_NO_PREV_DOC for the first)
  uint32_t doc_bits, tf_bits, count;
};

template <class L>
__device__ __forceinline__ BlkHdr blk_header(const uint8_t* blk) {
  const uint4 h = L::ld(reinterpret_cast<const uint4*>(blk));  // QwSkip: last_doc, prev_last_doc, byte_off, bits/count
  return BlkHdr{h.x, h.y, h.w & 0xFF, (h.w >> 8) & 0xFF, h.w >> 16};
}

// the lane's 4 values of a 4-lane-interleaved array of 128 values packed at `bits` (1..32) bits
template <class L>
__device__ __forceinline__ void unpack4(const uint4* p, uint32_t bits, uint32_t lane, uint32_t (&v)[4]) {
  const uint32_t bitpos = lane * bits, wi = bitpos >> 5, sh = bitpos & 31;
  const uint4 A = L::ld(p + wi);
  const uint4 B = (sh + bits > 32) ? L::ld(p + wi + 1) : make_uint4(0, 0, 0, 0);
  const uint32_t mask = 0xFFFFFFFFu >> (32 - bits);
  v[0] = __funnelshift_r(A.x, B.x, sh) & mask; v[1] = __funnelshift_r(A.y, B.y, sh) & mask;
  v[2] = __funnelshift_r(A.z, B.z, sh) & mask; v[3] = __funnelshift_r(A.w, B.w, sh) & mask;
}

// Doc ids of the lane's 4 postings, minus `ws` (mod 2^32; 0 gives absolute ids): strictly sorted deltas,
// doc[i] = doc[i-1] + v[i] + 1, summed by a warp inclusive scan from the previous block's last doc. Every lane of the
// warp must call it.
template <class L>
__device__ __forceinline__ void blk_docs(const uint8_t* blk, const BlkHdr& h, uint32_t ws, uint32_t lane, uint32_t (&doc)[4]) {
  uint32_t v[4] = {0, 0, 0, 0};
  if (h.doc_bits) unpack4<L>(reinterpret_cast<const uint4*>(blk + 16), h.doc_bits, lane, v);
  const uint32_t d0 = v[0] + 1, d1 = d0 + v[1] + 1, d2 = d1 + v[2] + 1, d3 = d2 + v[3] + 1;
  uint32_t incl = d3;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t n = __shfl_up_sync(0xFFFFFFFFu, incl, o);
    if ((int)lane >= o) incl += n;
  }
  const uint32_t basev = h.prev + (incl - d3) - ws;  // mod 2^32
  doc[0] = basev + d0; doc[1] = basev + d1; doc[2] = basev + d2; doc[3] = basev + d3;
}

// tfs of the lane's 4 postings (1 when the field keeps no frequencies)
template <class L>
__device__ __forceinline__ void blk_tfs(const uint8_t* blk, const BlkHdr& h, uint32_t lane, uint32_t (&tf)[4]) {
  tf[0] = tf[1] = tf[2] = tf[3] = 1;
  if (h.tf_bits) unpack4<L>(reinterpret_cast<const uint4*>(blk + 16) + h.doc_bits, h.tf_bits, lane, tf);
}

// Bm25Weight::score's tf / (tf + norm[fieldnorm id]) in f32 round-to-nearest. `tab` is float[256] norms, then
// float[QW_TFF_ROWS][256] quotients built with the same IEEE ops: tf below QW_TFF_ROWS reads the table.
__device__ __forceinline__ float tf_factor(const float* tab, uint32_t tf, uint32_t fn) {
  if (tf < QW_TFF_ROWS) return __ldg(tab + 256 + tf * 256 + fn);
  const float tff = (float)tf;
  return __fdiv_rn(tff, __fadd_rn(tff, __ldg(tab + fn)));
}

// Warp-cooperative 32-ary search of a skip list: the first index in [0, n) whose last_doc is >= doc (n if none), one
// round of coalesced loads per factor 32. All lanes return the same value.
__device__ __forceinline__ uint32_t first_block_ge(const QwSkip* skips, uint32_t n, uint32_t doc, uint32_t lane) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t step = (hi - lo + 31) / 32, idx = lo + lane * step;
    const bool before = idx < hi && __ldg(&skips[idx].last_doc) < doc;  // true for a prefix of the probes
    const uint32_t c = (uint32_t)__popc(__ballot_sync(0xFFFFFFFFu, before));
    if (c == 0) { hi = lo; break; }
    hi = min(hi, lo + c * step);
    lo = lo + (c - 1) * step + 1;
  }
  return lo;
}

}  // namespace qwk
