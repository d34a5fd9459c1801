// device_types.h — structures and value rules shared by the host (engine, aggregations) and the kernels.
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include "../../include/qwgpu.h"

#define QW_THREADS 512
#define QW_MIN_BLOCKS_PER_SM 2
#define QW_WARPS (QW_THREADS / 32)
#define QW_MAX_INSTR 96
#define QW_MAX_DCOLS 16                          /* columns a plan's query and sort may use */
#define QW_MAX_AGG_NODES QWGPU_MAX_AGG_NODES    /* aggregation nodes per plan */
#define QW_MAX_AGG_LEVELS QWGPU_MAX_AGG_LEVELS  /* nesting levels of a plan's aggregation tree (the hashed walk's stack) */
#define QW_MAX_AGG_COLS QWGPU_MAX_AGG_COLUMNS   /* columns first used by aggregation nodes, beyond QW_MAX_DCOLS */
#define QW_MAX_LEVELS QW_MAX_PLAN_DEPTH
#define QW_MAX_TERMS 64      /* TERM instructions per plan */
#define QW_BLK_TAB 160       /* staged blocks per (term, window) before falling back to direct mode */
#define QW_MAX_WBLK 512      /* staged blocks per window over all terms */
#define QW_HIST_BINS 2048    /* 11-bit radix digits */
#define QW_DIGIT_BITS 11
#define QW_KEY_BITS 192
#define QW_CAND_CAP 8192     /* candidates kept per split before the final sort (K <= QW_MAX_TOPK) */
#define QW_MAX_TOPK 4096     /* largest K that k_select sorts in one block (also the find_trace_ids limit) */
#define QW_MAX_HITS 20000    /* largest max_hits + start_offset of a request: the reference's 10 000 + 10 000 */
#define QW_SMEM_AGG_CELLS 4096

#ifdef __CUDACC__
#define QW_HOST_DEVICE __host__ __device__ __forceinline__
#else
#define QW_HOST_DEVICE static inline
#endif

// ---- tantivy MonotonicallyMappableToU64 (tantivy-columnar; SURVEY.md Appendix A.5) -------------
QW_HOST_DEVICE uint64_t i64_to_u64(int64_t v) { return (uint64_t)v ^ (1ull << 63); }
QW_HOST_DEVICE int64_t u64_to_i64(uint64_t v) { return (int64_t)(v ^ (1ull << 63)); }
// (the device takes the bit casts as intrinsics: a memcpy there compiles the aggregation walks differently)
QW_HOST_DEVICE uint64_t f64_to_u64(double d) {
#ifdef __CUDA_ARCH__
  const uint64_t bits = (uint64_t)__double_as_longlong(d);
#else
  uint64_t bits;
  memcpy(&bits, &d, 8);
#endif
  return (bits & (1ull << 63)) ? ~bits : (bits ^ (1ull << 63));
}
QW_HOST_DEVICE double u64_to_f64(uint64_t v) {
  const uint64_t bits = (v & (1ull << 63)) ? (v ^ (1ull << 63)) : ~v;
#ifdef __CUDA_ARCH__
  return __longlong_as_double((long long)bits);
#else
  double d;
  memcpy(&d, &bits, 8);
  return d;
#endif
}
// The f64 of a column's mapped value, as the stats, histogram and percentiles aggregations read it (ordinals of str
// and ip columns as numbers)
QW_HOST_DEVICE double qw_mapped_to_f64(uint32_t type, uint64_t m) {
  switch (type) {
    case QW_COL_U64: case QW_COL_BOOL: case QW_COL_STR: case QW_COL_IP: return (double)m;
    case QW_COL_I64: case QW_COL_DATETIME: return (double)u64_to_i64(m);
    default: return u64_to_f64(m);
  }
}
// Histogram position of a value: floor((val - offset) / interval), tantivy's bucket position before base_pos. The
// device fast paths find buckets through boundary tables the host builds with this formula, so both must share it.
QW_HOST_DEVICE double qw_hist_pos(double val, double offset, double interval) { return floor((val - offset) / interval); }
// Candidate capacity of a split whose plan asks for K hits: QW_CAND_CAP up to QW_MAX_TOPK (k_select's shared
// memory), above that 2K rounded up to a multiple of 1024 (the deep selection path, deep_select_kernel.cuh).
QW_HOST_DEVICE uint32_t qw_cand_cap(uint32_t K) { return K <= QW_MAX_TOPK ? (uint32_t)QW_CAND_CAP : (2u * K + 1023u) & ~1023u; }

// First work item of block b of a `grid`-block persistent launch over `total` items: block b walks the contiguous
// chunk [qw_chunk_begin(total, b, grid), qw_chunk_begin(total, b + 1, grid)).
QW_HOST_DEVICE uint32_t qw_chunk_begin(uint32_t total, uint32_t b, uint32_t grid) { return (uint32_t)(((uint64_t)total * b) / grid); }

// A strided threshold sample takes every stride-th item of each split (window; k_driver: posting block), starting at
// item s % stride of split s (at item 0 when stride is 1). Work item k of split s is its item qw_sample_item(k, s,
// stride); a split of n items has qw_sample_count(n, s, stride) work items. The host sizes the work list with the
// one and the kernels walk it with the other, so the two must agree.
QW_HOST_DEVICE uint32_t qw_sample_item(uint32_t k, uint32_t s, uint32_t stride) { return k * stride + (stride > 1 ? s % stride : 0u); }
QW_HOST_DEVICE uint32_t qw_sample_count(uint32_t n, uint32_t s, uint32_t stride) {
  const uint32_t phase = stride > 1 ? s % stride : 0u;
  return n > phase ? (n - phase + stride - 1) / stride : 0u;
}

// The flat (split, item) list a persistent launch walks
struct DWorkList {
  const uint32_t* first_work;  // prefix over splits of their (sampled) item counts; [n_splits + 1]
  uint32_t n_splits, total_work;
  uint32_t stride;             // threshold sample: every stride-th item (qw_sample_item; 1 = every item)
};

// The threshold sample of a BM25-union collect pass that samples itself (k_union<MODE_SAMPLE_COLLECT>): the first
// window of every block's chunk of the flat window list. first_work: prefix over the n splits of their windows
// ([n + 1]); max_hits: per split. True when the pass may run: at least 4 windows per block, and every split that
// has windows and asks for hits holds the first window of at least one block. Then stride[s] =
// max(1, floor(windows_s / samples_s)) is the weight of split s's sample (rounded down: a more conservative threshold).
static inline bool qw_fused_sample_plan(const uint32_t* first_work, const uint32_t* max_hits, uint32_t n, uint32_t grid, uint32_t* stride) {
  const uint32_t total = first_work[n];
  if (grid == 0 || total < 4ull * grid) return false;
  uint32_t b = 0;
  for (uint32_t s = 0; s < n; s++) {
    const uint32_t windows = first_work[s + 1] - first_work[s];
    uint32_t samples = 0;
    for (; b < grid && qw_chunk_begin(total, b, grid) < first_work[s + 1]; b++) samples++;
    if (windows && max_hits[s] && !samples) return false;
    stride[s] = samples ? (windows / samples > 1 ? windows / samples : 1u) : 1u;
  }
  return true;
}

enum { OP_TERM = 1, OP_RANGE = 2, OP_EXISTS = 3, OP_ALL = 4, OP_BOOL_BEGIN = 5, OP_BOOL_END = 6, OP_PHRASE = 7, OP_TERM_SET = 8,
       OP_COL_SET = 9 };

// The window program's plan limits: a plan whose lowering takes more TERM instructions or more instructions than this
// is refused. The query compiler asks the same question before it trades set groups for set nodes.
static inline bool qw_program_fits(uint64_t n_terms, uint64_t n_instr) { return n_terms <= QW_MAX_TERMS && n_instr <= QW_MAX_INSTR; }
enum { IF_SCORED = 1u, IF_HAS_TF = 2u, IF_HAS_FN = 4u, IF_BITS_FROM_SCORE = 8u };
#define QW_TFF_ROWS 16 /* tf-factor table: tff[tf][fieldnorm_id] = tf / (tf + norm[id]) for tf < 16 */

struct DInstr {  // 64 bytes
  uint32_t op, level, occur, flags;
  uint64_t a, b, c;  // TERM: data_off, widx_off, skip_off | RANGE: lo, hi | PHRASE: a = VBlk[] (device address), c = driver skip_off
                     // | TERM_SET: a = the node's doc bitmap (device address)
                     // | COL_SET: a = the split's sorted table of raw values (device address)
  uint32_t n;        // TERM: num_blocks   | BOOL_END: n_req | COL_SET: the table's length
  uint32_t m;        // TERM: win_shift    | BOOL_END: n_should
  uint32_t r;        // TERM: fn slot      | RANGE/EXISTS/COL_SET: column | BOOL_END: required_should
  float f;           // TERM: bm25 weight  | const-score leaves: boost
  uint32_t t;        // TERM: term slot (index among the plan's TERM instructions)
  uint32_t pad;
};

// A phrase evaluated by the pre-pass (phrase_kernel.cuh): one uncompressed posting block per 128-posting block of
// the phrase's driver term — doc = 0xFFFFFFFF where the driver posting's doc does not hold the phrase.
struct VBlk {
  uint32_t doc[QW_BLOCK_LEN];
  float val[QW_BLOCK_LEN];  // score contribution (0 when the phrase is not scored)
};
struct DPhraseTerm {
  uint64_t data_off, skip_off, pos_off, pidx_off;  // data-relative (QwImgTerm)
  uint32_t nblk, offset;                           // offset = position of the term inside the phrase
};
struct DPhrase {
  uint64_t data_base;  // the split's data region (device address)
  uint64_t out;        // VBlk[driver blocks] (device address)
  uint64_t fn_off;     // per-document fieldnorm ids, data-relative; ~0 = the field keeps none (constant id 1)
  uint64_t tab;        // the field's BM25 tables (device address): float[256] norms, then tff[16][256]
  float weight;        // (sum of the terms' idf) * (1 + K1) * boost
  uint32_t n_terms, driver, scored;
  uint32_t first_work;  // prefix of driver blocks over the batch's phrases
  uint32_t n_exp;       // phrase prefix: number of expansions of the last slot (0 = a plain phrase)
  uint64_t exp;         // phrase prefix: DPhraseTerm[n_exp]; phrase of more than QW_MAX_PHRASE_TERMS terms
                        // (k_phrase_long): DPhraseTerm[n_terms], the driver first, then by ascending doc_freq
                        // (device address; an index into the plan's, then the batch's records until Run::stage)
  DPhraseTerm t[QW_MAX_PHRASE_TERMS];  // up to QW_MAX_PHRASE_TERMS terms (phrase prefix: the n_terms exact terms)
};

// A term-set node evaluated by the pre-pass (termset_kernel.cuh) into a doc bitmap of ceil(num_docs / 32) words.
struct DTermSetNode {
  uint64_t bitmap;  // device address
};
// Lowering numbers `node` within the plan; Run::lay_out renumbers it within the batch and sets `first_block`.
struct DTermSetTerm {
  uint64_t data, skip;  // the term's posting blocks and skip list (device addresses)
  uint32_t nblk;        // its posting blocks
  uint32_t first_block; // prefix of nblk over the batch's term-set terms (the pre-pass's flat block list)
  uint32_t node;        // DTermSetNode of the batch
  uint32_t pad;
};

struct DCol {  // 48 bytes
  uint64_t values_off, index_off, min_value, gcd;
  uint32_t bits, card, type, nwords64;
};

struct DAgg {
  uint32_t kind, parent, first_child, num_children;
  uint32_t col, num_buckets, has_bounds, num_ranges;
  uint32_t has_missing, cell_base;
  uint32_t is_f64;  // STATS: 1 = sum doubles, 0 = the exact u64 sum of raw offsets (qw_stats_sum_exact, host-decided)
  uint32_t comp;    // TERMS / HISTOGRAM: QW_AGG_COMP_* flags (QwAggNode.reserved), read by the hashed walk only
  double interval, offset, bound_min, bound_max;
  int64_t base_pos;
  // fast path (flat bucket aggregations over single-valued columns, see lower_aggs): histogram
  // buckets are found in RAW space — bounds[k] = smallest bit-packed raw value that falls into
  // bucket >= k (k = 0..num_buckets), computed on the host with the reference f64 formula
  // (common.h hist_bounds), so the device needs no f64 arithmetic and stays bit-exact
  uint64_t bounds;       // device address of uint64[num_buckets + 1] (HISTOGRAM only)
  float inv_step;        // ~ num_buckets / (bounds[nb] - bounds[0]): first guess of the bucket
  uint32_t stat_base;    // STATS on the fast path: first of this node's {sum, ~min, max} triples in shared memory
  uint64_t comp_after;   // composite source: the split's `after` bound (QwAggNode.range_from[0]); keeps sizeof(DAgg) a
                         // multiple of 16 (copied to shared memory as uint4)
  uint64_t range_from[QW_MAX_AGG_RANGES], range_to[QW_MAX_AGG_RANGES];
};
static_assert(sizeof(DInstr) % 16 == 0 && sizeof(DCol) % 16 == 0 && sizeof(DAgg) % 16 == 0, "uint4-copied structs");

// Composite sort key: a big-endian bit string of at most 192 bits, greater = better, packed from the
// most significant bit with no padding between fields:
//   [has1:1][r1:rbits0] [has2:1][r2:rbits1] [doc':doc_bits]
// r_i is the RANK of sort value i: the column's bit-packed raw value (raw_max - raw for ascending
// order), or for _score a value-linear 10-bit bucket followed by the order-preserving f32 bits (42
// bits as first key, 32 as second). A field that cannot discriminate (doc-id sort, column absent from
// the split) contributes no bits at all. doc' is the doc id (complemented within doc_bits when the
// first order is ascending). This is exactly the total order of SegmentPartialHitSortingKey
// (quickwit-search/src/collector.rs:1082-1112), None last; because the fields are only as wide as
// the split's data needs, every 11-bit radix digit of the key discriminates.
struct alignas(16) DKeySpec {
  uint32_t kind[2], order[2], col[2];
  uint32_t rbits[2];     // width of r_i
  uint32_t hasbit[2];    // 1: a has-value bit precedes r_i
  uint32_t doc_bits, total_bits;
  uint32_t top_mode;     // how the first 11 key bits are derived cheaply (QW_TOP_*)
  float score_scale;     // SCORE: lin = min(1023, (uint)(score * scale))
  uint64_t raw_max[2];   // r_i = order == DESC ? raw : raw_max - raw
  // total_bits <= 64 (the usual case): the key is w0 = OR of (field << shift), shifts precomputed
  uint32_t narrow, sh_has[2], sh_r[2], sh_doc;
};
static_assert(sizeof(DKeySpec) % 16 == 0, "uint4-copied struct");
enum { QW_TOP_FULL = 0, QW_TOP_SCORE = 1, QW_TOP_COLUMN = 2, QW_TOP_DOC = 3 };

struct DThresh {  // per split, device-resident, written by k_pick
  uint64_t key[3];       // candidates are docs with composite key >= key
  uint32_t prefix_bits;  // number of leading bits of `key` that are fixed so far
  uint32_t above;        // docs strictly above the prefix (exact path bookkeeping)
  uint32_t done;         // 1 when the candidate set fits qw_cand_cap(K)
  uint32_t matched;      // docs matching the prefix at the last level
};

struct DSplitPlan {
  uint64_t data_base;  // device address of the split's data region
  uint32_t num_docs, num_windows;
  uint32_t n_instr, instr_base;
  uint32_t n_cols, col_base;
  uint32_t n_aggs, agg_base;
  uint32_t n_terms, n_levels;
  uint32_t max_hits, scoring;
  uint32_t n_fn_slots, n_cells;
  uint32_t fused_score_root;  // root bool is a pure OR of positive-weight scored terms
  uint32_t fast_aggs;         // every aggregation is a bucket aggregation (optionally with stats children)
                              // or a stats node over always-present single-valued columns
  uint32_t n_stat_cells;   // fast path: number of privatised stats cells
  uint32_t score_hits;     // k_select writes QwScoreHit records (qw_plan_score_hits; never in a merged batch)
  uint64_t fn_off[2];      // data-relative fieldnorm arrays staged per window
  uint64_t bm25_tab[2];    // device addresses of float[256] BM25 norm tables, followed by the
                           // float[QW_TFF_ROWS][256] tf-factor table of the same field
  DKeySpec key;
  QwSearchAfter sa;
  uint64_t out_num_hits;   // device address of a uint64 counter
  uint64_t out_hist;       // device address of uint32[QW_HIST_BINS]
  uint64_t out_cand_count; // device address of a uint32 counter
  uint64_t out_cands;      // device address of uint64[3 * qw_cand_cap(max_hits)]
  uint64_t out_cells;      // device address of QwAggCell[n_cells]
  uint64_t out_hits;       // device address of QwHit[max_hits] (score_hits: QwScoreHit[max_hits])
  uint64_t out_nhits;      // device address of uint32 (hits written by k_select)
  // find_trace_ids (trace_kernel.cuh); tr_on == 0 when the plan has no QW_AGG_TRACE_IDS node
  uint64_t tr_best;        // device address of uint64[tr_num_ords]: latest span per trace ordinal (0 = none)
  uint64_t match_out;      // 0, or the device address of uint32[ceil(num_docs / 32)] where k_window's collect pass
                           // writes every window's final match words: the find_trace_ids replay's input, or the
                           // predicate-cache entry that a fill plan fills
  uint64_t tr_state;       // device address of a DTraceState
  uint64_t tr_tie;         // device address of a uint32 in the split's output header: 1 = the replay ran
  uint32_t tr_on, tr_n;    // N = num_traces
  uint32_t tr_num_ords;    // entries of tr_best (the column dictionary's size, at least 1)
  uint32_t tr_ord_col, tr_ts_col;  // DCol indices of the trace-id and timestamp columns (ts: 0xFFFFFFFF = absent)
  // hashed aggregation cells (qw_agg_hashed; kernels.cuh agg_collect_hashed); hashed == 0 for dense plans
  uint32_t hashed;
  uint32_t h_cap;          // cell capacity of this run
  uint32_t h_mask;         // table slots - 1 (slots: a power of two >= h_cap)
  uint64_t h_table;        // device address of uint32[slots]: cell id, QW_HSLOT_EMPTY / _BUSY / _FULL
  uint64_t h_keys;         // device address of DHKey[h_cap]
  uint64_t h_cells;        // device address of QwAggCell[h_cap]
  uint64_t h_ctr;          // device address of a uint32 in the split's output header: cells claimed | overflow << 31
};
// key record of a hashed cell (the rest of its QwAggEntry)
struct DHKey {
  uint64_t key;
  uint32_t node_flags;  // node | QwAggEntry.flags << 8
  uint32_t parent;
};
#define QW_HSLOT_EMPTY 0xFFFFFFFFu
#define QW_HSLOT_BUSY 0xFFFFFFFEu
#define QW_HSLOT_FULL 0xFFFFFFFDu

static_assert(offsetof(DSplitPlan, key) % 16 == 0 && sizeof(DSplitPlan) % 16 == 0, "DKeySpec is read as uint4");

// The head of a split's region in the call's output buffer; the split's hit list and aggregation cells follow it
struct DSplitOut {
  uint64_t num_hits;       // matching docs (out_num_hits)
  uint64_t eligible;       // docs eligible for the top-K (out_num_hits + 1)
  uint32_t n_hits;         // hits written by k_select (out_nhits)
  uint32_t cand_count;     // candidates of the collect pass (out_cand_count)
  uint32_t trace_replayed; // 1: k_trace_replay ran (tr_tie)
  uint32_t hashed_cells;   // hashed cells claimed | overflow << 31 (h_ctr)
};
static_assert(sizeof(DSplitOut) == 32 && offsetof(DSplitOut, eligible) == 8 && offsetof(DSplitOut, n_hits) == 16 && offsetof(DSplitOut, cand_count) == 20 &&
              offsetof(DSplitOut, trace_replayed) == 24 && offsetof(DSplitOut, hashed_cells) == 28, "split output header");

// One hit of a device merge (k_merge): split = the list it came from, or the global split rank of a cross-rank merge
struct MergedHit {
  QwHit hit;
  uint32_t split, pad;
};
// A device-merged list is [RankHeader][MergedHit x k]: the batch's merge (a rank's gather record) and the cross-rank
// merge alike. k_merge writes n_hits; k_rank_header fills in a gather record the sums the root merge adds up
// (collector.rs:914-974): num_hits over the batch's splits, split accounting from the host.
struct RankHeader {
  uint32_t n_hits, pad;
  uint64_t num_hits, attempted, successful, n_failed, reserved[3];
};
static_assert(sizeof(MergedHit) == sizeof(QwHit) + 8 && sizeof(RankHeader) == 64, "merge records");

struct SmemLevel {
  uint32_t req, shd, nt, cnt, msum, ssum;  // byte offsets; 0xFFFFFFFF = not allocated
  uint32_t rsc, pad;                       // result score array of the level (msum, else ssum)
};
struct SmemLayout {
  uint32_t instr, cols, aggs, key, hitq;  // hitq: per-warp compacted hit queues of the generic collect
  uint32_t rangeq;  // per-warp queues of required RANGE / EXISTS clauses (0xFFFFFFFF: probe per bitmap word)
  SmemLevel lvl[QW_MAX_LEVELS];
  uint32_t tmp, fn[2];          // scratch bitmap; staged fieldnorm bytes per scored field
  uint32_t rng, blkrec, termblk, stage, hist, misc;  // hist aliases stage (dead by collect time)
  uint32_t l0hist;  // COLLECT pass: exact level-0 digit histogram of the window's matches (0xFFFFFFFF: not recorded)
  uint32_t total;
};

struct KParams {
  const DSplitPlan* plans;
  const DInstr* instrs;
  const DCol* cols;
  const DAgg* aggs;
  DThresh* thresh;
  DWorkList wl;      // (split, window) list; sampled passes: the sampled windows
  uint32_t W;        // window size in docs (<= 32768; a power of two, except 15360 in BM25-union batches)
  uint32_t level;    // MODE_HIST: radix level being histogrammed
  uint32_t use_prefix;  // MODE_HIST: restrict to docs whose key matches thresh prefix
  uint32_t smem_aggs;   // 1: aggregation counts privatised in shared memory
  uint32_t stage_bytes; // capacity of the posting staging area
  // second-chance top-K (engine.cu): a COLLECT pass may record the exact level-0 histogram and each
  // window's best level-0 digit; refinement passes then skip verified splits and windows that cannot
  // hold a candidate, and only emit candidates (hit counts / aggregations are already final)
  uint32_t rec_l0;        // COLLECT: record out_hist + wmax
  uint32_t refine;        // 1: skip splits with split_state == 0 and windows with wmax < threshold digit
  uint32_t cands_only;    // COLLECT: emit candidates only
  uint16_t* wmax;         // per flat window: 1 + best level-0 digit among its matches (0: no match)
  const uint32_t* split_state;  // per split: 1 = needs refinement
  const uint32_t* sample_win;   // sampled passes: per work item, window | edge << 31 (null: strided formula)
  SmemLayout sm;
};
