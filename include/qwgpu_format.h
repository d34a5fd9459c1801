/*
 * qwgpu_format.h — plain-old-data layouts shared across the C ABI of libqwgpu:
 *   (1) the split IMAGE (what a registered split looks like in host memory / HBM),
 *   (2) the per-split search PLAN (seam C of SURVEY.md §3.4: what replaces
 *       `searcher.search(&query, &collector)` at quickwit-search/src/leaf.rs:637),
 *   (3) the per-split RESULT (the fields of `LeafSearchResponse` produced by
 *       `QuickwitSegmentCollector::harvest`, quickwit-search/src/collector.rs:564-594).
 *
 * Everything is little-endian, naturally aligned, no pointers — only byte offsets — so the same
 * bytes can be mmapped, sent over FFI from Rust (`#[repr(C)]`), or copied to the device verbatim.
 *
 * The image follows the SHAPES of a tantivy segment (SURVEY.md Appendix A: 128-doc bit-packed
 * posting blocks with 4-lane interleave + skip entries, 1-byte fieldnorm ids, bit-packed columns
 * with min/gcd header, dictionary-encoded string columns), but it is OUR format: tantivy's byte
 * layout is not pinned by anything in the reference repository (SURVEY.md §8c "NOT pinned").
 */
#ifndef QWGPU_FORMAT_H
#define QWGPU_FORMAT_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define QW_IMG_MAGIC 0x31474D4947575151ull /* "QQWGIMG1" */
#define QW_IMG_VERSION 3u
#define QW_BLOCK_LEN 128u                  /* tantivy COMPRESSION_BLOCK_SIZE */
#define QW_TERMINATED 0x7FFFFFFFu          /* tantivy TERMINATED sentinel (i32::MAX as u32) */
#define QW_NO_PREV_DOC 0xFFFFFFFFu
#define QW_MIN_WIN_SHIFT 12u /* index windows are >= 4096 docs; an evaluation window (<= 8192 docs) spans <= 2 entries */

/* ---------------------------------------------------------------- image ---------------------- */

typedef struct QwImgHeader {
  uint64_t magic;
  uint32_t version;
  uint32_t num_docs;
  uint32_t num_fields;  /* inverted (text) fields */
  uint32_t num_terms;   /* dictionary entries over all fields, sorted by (field_id, bytes) */
  uint32_t num_columns; /* fast fields */
  uint32_t reserved0;
  uint64_t fields_off;     /* QwImgField[num_fields] */
  uint64_t terms_off;      /* QwImgTerm[num_terms]   */
  uint64_t term_bytes_off; /* concatenated term bytes */
  uint64_t term_bytes_len;
  uint64_t columns_off; /* QwImgColumn[num_columns] */
  uint64_t strings_off; /* names + column dictionaries (host-only blob) */
  uint64_t strings_len;
  uint64_t data_off; /* device-resident region: postings, skip lists, fieldnorms, column data */
  uint64_t data_len; /* multiple of 16 */
  uint64_t total_len;
  uint64_t reserved1[3];
} QwImgHeader; /* 128 bytes */

enum { QW_FIELD_HAS_FREQS = 1u, QW_FIELD_HAS_FIELDNORMS = 2u, QW_FIELD_HAS_POSITIONS = 4u };
/* QW_TOK_IP: an indexed `type: ip` field; its terms are 16-byte big-endian IPv6 addresses (as QW_COL_IP's dictionary),
 * recorded `basic` without fieldnorms. Query text is parsed as one address, never tokenized. */
enum { QW_TOK_RAW = 0u, QW_TOK_DEFAULT = 1u, QW_TOK_IP = 2u };

typedef struct QwImgField {
  uint32_t name_off, name_len; /* into strings blob */
  uint32_t flags;              /* QW_FIELD_* */
  uint32_t tokenizer;          /* QW_TOK_* */
  uint64_t total_num_tokens;   /* Σ field lengths; average_fieldnorm = total / num_docs */
  uint64_t fieldnorm_off;      /* data-relative; num_docs bytes (fieldnorm ids); valid iff HAS_FIELDNORMS */
  uint32_t first_term, num_terms;
  uint64_t reserved;
} QwImgField; /* 48 bytes */

typedef struct QwImgTerm {
  uint32_t field_id;
  uint32_t bytes_off, bytes_len; /* into term bytes blob */
  uint32_t doc_freq;
  uint32_t num_blocks; /* ceil(doc_freq / 128) */
  uint32_t win_shift;  /* window index granularity: one entry per 2^win_shift docs (>= 12) */
  uint64_t skip_off; /* data-relative: QwSkip[num_blocks] (CPU-style seek structure) */
  uint64_t data_off; /* data-relative: blocks, each [QwSkip header][packed docs][packed tfs][fieldnorm ids] */
  uint64_t data_len;
  uint64_t widx_off; /* data-relative: QwWinIdx[ceil(num_docs / 2^win_shift)] */
  uint64_t tf_len;   /* bytes of data_len that are packed term frequencies (roofline accounting) */
  uint64_t fn_len;   /* bytes of data_len that are per-posting fieldnorm ids (128 per block, see QwSkip) */
  uint64_t sub_off;  /* data-relative: QwSubIdx[num_blocks] (doc-id checkpoints inside each block) */
  /* positions (fields indexed with `record: position`, QW_FIELD_HAS_POSITIONS; both 0 otherwise): the token
   * positions of every posting, in posting order — posting i owns tf[i] consecutive entries, ascending
   * (tantivy's .pos stream keeps them delta-bit-packed per 128 positions; here they are plain uint32) */
  uint64_t pos_off;  /* data-relative: uint32 positions[sum of tf] */
  uint64_t pidx_off; /* data-relative: uint32 first_pos[num_blocks + 1] — index into positions[] of the first
                        position of each block; [num_blocks] = sum of tf */
} QwImgTerm; /* 96 bytes */

/* Window index: for index-window j (docs [j<<win_shift, (j+1)<<win_shift)) the byte range
 * [start, end) of QwImgTerm data holding every block that overlaps it (start == end if none).
 * This is what lets a GPU thread block that owns a doc-id window fetch exactly the posting bytes
 * it needs with ONE dependent load instead of a binary search over the skip list. */
typedef struct QwWinIdx {
  uint32_t start, end;             /* byte range inside QwImgTerm data */
  uint32_t first_block, end_block; /* the same blocks as ordinals into the skip list */
} QwWinIdx;

/* One skip entry per posting block; 16 bytes = one coalesced 128-bit load.
 * A block holds `count` (1..128) postings. Doc ids are stored as strictly-sorted deltas:
 *   v[i] = doc[i] - doc[i-1] - 1, with doc[-1] := prev_last_doc (0xFFFFFFFF for the first block,
 *   arithmetic mod 2^32), bit-packed at `doc_bits` bits with the BitPacker4x interleave
 *   (value i lives in lane i%4 at position i/4; 128-bit word w holds 32-bit word w of the four
 *   lanes) => 16*doc_bits bytes. Term frequencies follow, raw, at `tf_bits` bits => 16*tf_bits
 *   bytes (tf_bits == 0 when the field is indexed `record: basic`; tf := 1).
 * When the field has fieldnorms, 128 bytes follow: the fieldnorm id of each posting's document
 * (byte i = fieldnorm id of doc[i], zero padded). tantivy keeps fieldnorms per document only; the
 * image ALSO keeps that array (QwImgField.fieldnorm_off) but denormalises the id next to every
 * posting so that BM25 scoring reads one contiguous byte stream per block instead of a random
 * 1-byte gather per posting (the bytes read equal SURVEY.md 8d's "1 B per scored posting").
 * The trailing partial block uses the same layout, zero padded (tantivy VInt-encodes it; a
 * real-split ingester transcodes, SURVEY.md §8f-2). */
typedef struct QwSkip {
  uint32_t last_doc;
  uint32_t prev_last_doc;
  uint32_t byte_off; /* of this block's inline header, relative to QwImgTerm.data_off */
  uint8_t doc_bits;
  uint8_t tf_bits;
  uint16_t count;
} QwSkip;

/* Checkpoints inside a posting block: the doc id reached after 32, 64 and 96 postings, relative to
 * prev_last_doc (mod 2^32), and the block's whole span. A reader that only needs the postings of a
 * doc-id sub-range can start decoding at any 32-posting boundary (sub-block s starts from
 * prev_last_doc + ck[s-1]) instead of prefix-summing the block from its beginning — the GPU union
 * kernel gives every warp its own doc-id range of a window and decodes only the sub-blocks that
 * overlap it. Sub-blocks past `count` are empty and repeat `span`. */
typedef struct QwSubIdx {
  uint32_t ck[3]; /* doc[32k - 1] - prev_last_doc for k = 1..3 (span when 32k > count) */
  uint32_t span;  /* last_doc - prev_last_doc */
} QwSubIdx;

enum {
  QW_COL_U64 = 0,
  QW_COL_I64 = 1,
  QW_COL_F64 = 2,
  QW_COL_BOOL = 3,
  QW_COL_DATETIME = 4, /* i64 nanoseconds, truncated to fast_precision at build time */
  QW_COL_STR = 5,      /* term ordinals into a sorted dictionary */
  QW_COL_BYTES = 6,    /* `type: bytes` fast field: ordinals into a sorted dictionary of raw byte strings, stored like
                          QW_COL_STR (dict_off / dict_num_terms). Only the find_trace_ids collector reads it; queries,
                          sorts and aggregations on it are refused. */
  QW_COL_IP = 7        /* `type: ip` fast field: ordinals into a sorted dictionary of 16-byte big-endian IPv6 addresses
                          (an IPv4 address as its IPv4-mapped form ::ffff:a.b.c.d), stored like QW_COL_STR. Byte order
                          is numeric order, so the compiler turns every equality and range on an address into an
                          ordinal range per split; the device only ever sees ordinals. Sorting on it is refused, and
                          only `terms` aggregates it. */
};
enum { QW_CARD_FULL = 0, QW_CARD_OPTIONAL = 1, QW_CARD_MULTI = 2 };

/* Column values are stored in tantivy's order-preserving u64 mapping
 * (MonotonicallyMappableToU64: i64 -> x ^ 1<<63, f64 -> sign-flip trick, bool -> 0/1,
 * DateTime -> i64 nanos, Str -> ordinal) as raw = (mapped - min_value) / gcd, bit-packed
 * little-endian at `bits` bits per value (value i occupies bits [i*bits, (i+1)*bits)).
 * index (data-relative):
 *   FULL:     none; value index == doc id.
 *   OPTIONAL: uint64 present[ceil(num_docs/64)] then uint32 rank[ceil(num_docs/64)+1]
 *             (rank[w] = number of set bits before word w); value index = rank + popc(below).
 *   MULTI:    uint32 start[num_docs+1]; values of doc d are [start[d], start[d+1]). */
typedef struct QwImgColumn {
  uint32_t name_off, name_len;
  uint32_t type;        /* QW_COL_* */
  uint32_t cardinality; /* QW_CARD_* */
  uint64_t min_value, max_value, gcd;
  uint64_t num_vals;
  uint32_t bits;
  uint32_t dict_num_terms; /* STR only */
  uint64_t values_off, values_len; /* data-relative; padded with 16 zero bytes */
  uint64_t index_off, index_len;   /* data-relative */
  uint64_t dict_off, dict_len;     /* strings-blob relative: uint32 offs[n+1] then bytes */
  uint64_t reserved;
} QwImgColumn; /* 112 bytes */

/* ---------------------------------------------------------------- plan ----------------------- */

#define QW_PLAN_MAGIC 0x4E4C5051u /* "QPLN" */
#define QW_MAX_PLAN_DEPTH 4
#define QW_MAX_PHRASE_TERMS 8 /* exact terms of one PHRASE_PREFIX node (plus one); PHRASE nodes above it run the
                                 long-phrase pre-pass */
#define QW_MAX_PHRASE_LEN 256 /* TERM children of one PHRASE node */
#define QW_MAX_PREFIX_EXPANSIONS 1024 /* expansion children of one PHRASE_PREFIX node */
#define QW_MAX_SET_TERMS 65536 /* children of one TERM_SET or COL_SET node */

enum {
  QW_NODE_TERM = 1,   /* tantivy TermQuery */
  QW_NODE_RANGE = 2,  /* tantivy FastFieldRangeQuery; const score 1 */
  QW_NODE_BOOL = 3,   /* tantivy BooleanQuery */
  QW_NODE_ALL = 4,    /* AllQuery; score 1 */
  QW_NODE_NONE = 5,   /* EmptyQuery */
  QW_NODE_EXISTS = 6, /* ExistsQuery on a column; const score 1 */
  QW_NODE_PHRASE = 7, /* tantivy PhraseQuery, slop 0: children = its TERM nodes in phrase order, all of one field
                         with positions, 2 <= children <= QW_MAX_PHRASE_LEN; child k's `lo` = position offset of
                         the term inside the phrase, any values (tantivy PhraseQuery::new_with_offset: gapped,
                         starting above 0, not ascending) whose spread max - min is below 2^31. A doc matches when
                         its positions align: some integer c, which may be negative, has term k at c + lo_k for
                         every k; phrase_count = number of such c. Score = bm25_weight * tf-factor(phrase_count, fieldnorm) with
                         bm25_weight = (sum of the terms' idf, duplicates included) * (1 + K1) * boost
                         (Bm25Weight::for_terms). */
  QW_NODE_PHRASE_PREFIX = 8, /* tantivy PhrasePrefixQuery with at least one exact term: children = the k exact TERM
                               nodes in phrase order, then the E expansion TERM nodes of the last slot (the field's
                               first max_expansions terms, in byte order, that start with the prefix); the node's
                               `lo` = k; each child's `lo` = its position offset, so every expansion carries the last
                               offset. All of one field with positions; 1 <= k < QW_MAX_PHRASE_TERMS,
                               1 <= E <= QW_MAX_PREFIX_EXPANSIONS; offsets as in QW_NODE_PHRASE. A doc matches when
                               its positions align: some integer c, which may be negative, has exact term i at
                               c + lo_i for every i and some expansion at c + lo_last. Never scored: the
                               node is only valid where its score is not read (filter / must_not, or any sort
                               other than _score). */
  QW_NODE_TERM_SET = 9, /* a set of terms (tantivy AutomatonWeight of a regex query): children = E TERM nodes of one
                          field with strictly increasing term_ord, 1 <= E <= QW_MAX_SET_TERMS. A doc matches when it holds
                          any child. Positions are not needed, and the children do not count toward the plan's TERM
                          clauses. Never scored: the node is only valid where its score is not read (filter / must_not,
                          or any sort other than _score). */
  QW_NODE_CACHE = 10, /* the reference's CacheNode (quickwit-query/src/query_ast/cache_node.rs): exactly one child, the
                        inner subtree, matching the same docs. A context with a predicate cache
                        (qwgpu_set_predicate_cache_budget) keeps the child's doc set per split and reads it instead of
                        evaluating the child again. Never scored: in a scoring clause of a query ranked by _score, with
                        the cache disabled, or around ALL / NONE, the engine lowers it as its child. */
  QW_NODE_COL_SET = 11 /* a set of values of one fast column (tantivy TermSetQuery / a bool of term queries on a
                          fast-only field): the node's `column` = the column; children = E RANGE nodes on that column,
                          each with lo == hi in mapped-u64 space, strictly increasing, 1 <= E <= QW_MAX_SET_TERMS. A doc
                          matches when any of its values equals a child's. Never scored, like QW_NODE_TERM_SET. */
};
enum { QW_OCCUR_MUST = 0, QW_OCCUR_SHOULD = 1, QW_OCCUR_MUST_NOT = 2, QW_OCCUR_FILTER = 3 };

/* Children of a BOOL node are the nodes [first_child, first_child + num_children) in the node
 * array, each tagged with its `occur`. FILTER = Must(ConstScoreQuery(q, 0.0))
 * (quickwit-query/src/query_ast/tantivy_query_ast.rs:345-377). */
typedef struct QwPlanNode {
  uint32_t kind;
  uint32_t occur; /* role in the parent BOOL (ignored for the root) */
  float boost;    /* multiplies the node's score (QueryAst::Boost); 1.0 by default */
  uint32_t first_child, num_children;
  uint32_t min_should_match; /* BOOL; 0xFFFFFFFF = unset */
  /* TERM */
  uint32_t term_ord;  /* index into QwImgTerm[]; 0xFFFFFFFF = term absent from the split */
  uint32_t field_id;
  float bm25_weight;  /* idf * (1 + K1), already including boost; host-computed (f32) */
  /* RANGE / EXISTS */
  uint32_t column;  /* index into QwImgColumn[]; 0xFFFFFFFF = column absent */
  uint64_t lo, hi;  /* inclusive bounds in the column's mapped-u64 space */
} QwPlanNode; /* 56 bytes */

enum { QW_SORT_NONE = 0, QW_SORT_DOCID = 1, QW_SORT_SCORE = 2, QW_SORT_COLUMN = 3 };
enum { QW_ORDER_ASC = 0, QW_ORDER_DESC = 1 }; /* quickwit SortOrder: ASC=0, DESC=1 */

typedef struct QwSortSpec {
  uint32_t kind;   /* QW_SORT_* (QW_SORT_NONE only valid for the second key) */
  uint32_t order;  /* QW_ORDER_* */
  uint32_t column; /* QW_SORT_COLUMN: column index, 0xFFFFFFFF = missing (all None) */
  uint32_t reserved;
} QwSortSpec;

/* search_after, already converted to the u64 fast-field space
 * (SearchAfterSegment::new, quickwit-search/src/top_k_collector.rs:829-872). */
typedef struct QwSearchAfter {
  uint32_t present;
  uint32_t has_v1, has_v2;
  uint32_t compare_on_equal; /* !search_after.split_id.is_empty() */
  int32_t precomp_order;     /* order1.compare(split_id, sa.split_id).then(segment_ord): -1/0/1 */
  uint32_t doc_id;
  uint64_t v1, v2;
} QwSearchAfter;

enum {
  QW_AGG_TERMS = 1,
  QW_AGG_HISTOGRAM = 2,      /* also date_histogram (interval/offset pre-scaled to column units) */
  QW_AGG_RANGE = 3,
  QW_AGG_STATS = 4,          /* stats / avg / sum / min / max / value_count share one collector. With `has_missing`
                                (`missing_value` = the f64 bits of the `missing` value, which the device never reads)
                                the node also counts, under every parent bucket, the matched docs without a value in
                                its column (every matched doc when the split lacks the column): the entry with
                                QW_AGG_ENTRY_MISSING (key 0) next to the node's cell, or in the dense layout a second
                                bank of cells after the first. The host folds count * missing into the metric. */
  QW_AGG_TRACE_IDS = 5,      /* FindTraceIdsCollector (quickwit-search/src/find_trace_ids_collector.rs): the only node
                                of its plan. `column` = the trace-id QW_COL_BYTES column, `reserved` = the span timestamp
                                column (0xFFFFFFFF when absent from the split: every timestamp reads 0),
                                `num_buckets` = num_traces (N). Its N cells hold the split's result in no particular
                                order: cell j is a span when `count` == 1, with `sum_bits` = the trace id's
                                ordinal in the column dictionary and `max_mapped` = the span timestamp in the
                                order-preserving i64 mapping. */
  QW_AGG_PERCENTILES = 6     /* percentiles (a metric: no children). `column` = the value column; `num_buckets` = the bins
                                of the split's DDSketch boundary table for that column (quickwit_b200/csrc/ddsketch.h:
                                every bin between those of the column's minimum and maximum, in value order), plus one
                                when `has_missing`; `missing_value` = the f64 bits of the `missing` value. A plan that
                                holds one always takes the hashed layout (qw_agg_hashed). Its entries: key = the bin's
                                index in that table (indices increase with the value: negative store, zero count,
                                positive store), cell.count = the values in the bin, min_mapped / max_mapped = their
                                smallest / largest value in the column's mapped space, sum_bits = 0; a matched doc
                                without a value counts once in the entry with QW_AGG_ENTRY_MISSING (key 0) when
                                `has_missing`, and nowhere otherwise. */
};

#define QW_MAX_AGG_RANGES 16

/* Composite aggregation (DESIGN.md §4.4, composite): a composite with sources s1..sn lowers to a chain of n
 * QW_AGG_TERMS / QW_AGG_HISTOGRAM nodes, each the only child of the one before, with the composite's
 * sub-aggregations below the last. Each source node carries the composite descriptor in fields its kind does not
 * use:
 *   reserved      = QW_AGG_COMP_* flags (0 on every node that is not a composite source);
 *   range_to[0]   = the composite's `size`;
 *   range_from[0] = the split's bound for the `after` value of this source, in the node's key space (TERMS: the
 *                   bit-packed raw value, HISTOGRAM: the bucket index relative to base_pos): with ascending order
 *                   the smallest key that is not before `after`, with descending order the largest; EXACT when
 *                   that key equals `after`, AFTER_ALL when every key of the split comes before it.
 * A `missing_bucket` source sets has_missing; on a HISTOGRAM node the missing bucket is the last of num_buckets
 * and its entries carry QW_AGG_ENTRY_MISSING, as on TERMS. The walk keeps a key of a composite level only when its
 * path is not before the `after` tuple; HAS_AFTER is cleared on every level when a split cannot place `after` in
 * its key spaces (the host filters then, and AFTER_HOST is set). After the walk, k_composite_cut keeps each
 * composite's first `size` leaves with their chains and sub-aggregation entries (composite_kernel.cuh). */
enum {
  QW_AGG_COMP_LEVEL = 1u,      /* the node is a source of a composite aggregation */
  QW_AGG_COMP_LAST = 2u,       /* the last source of its composite */
  QW_AGG_COMP_DESC = 4u,       /* `order: desc` (null last; ascending order puts null first) */
  QW_AGG_COMP_MISSING = 8u,    /* `missing_bucket: true` */
  QW_AGG_COMP_HAS_AFTER = 16u, /* filter this level against range_from[0] */
  QW_AGG_COMP_AFTER_NULL = 32u,/* the `after` value of this source is null */
  QW_AGG_COMP_EXACT = 64u,     /* range_from[0] is `after` itself */
  QW_AGG_COMP_AFTER_ALL = 128u, /* every non-null key of the split comes before `after` */
  QW_AGG_COMP_AFTER_HOST = 256u /* the request has `after` but the walk does not filter (HAS_AFTER cleared): the
                                   device does not cut the composite either, the host filters and cuts */
};
#define QW_AGG_COMP_MAX_SIZE 65000u /* the reference's default aggregation_bucket_limit */

/* One aggregation node. Bucket aggregations may have children (sub-aggregations):
 * nodes [first_child, first_child+num_children). Top-level aggs have parent == 0xFFFFFFFF. */
typedef struct QwAggNode {
  uint32_t kind;
  uint32_t parent;
  uint32_t first_child, num_children;
  uint32_t column;      /* 0xFFFFFFFF = column absent in this split */
  uint32_t num_buckets; /* dense bucket space of this node in this split (host-computed) */
  /* HISTOGRAM: bucket_pos = floor((val_f64 - offset) / interval) (all in column units, f64);
   * dense index = bucket_pos - base_pos. */
  double interval, offset;
  int64_t base_pos;
  /* hard_bounds (inclusive, f64 in column units); has_bounds=0 when absent */
  uint32_t has_bounds;
  uint32_t num_ranges;
  double bound_min, bound_max;
  /* RANGE: bucket i = [range_from[i], range_to[i]) in mapped-u64 space */
  uint64_t range_from[QW_MAX_AGG_RANGES], range_to[QW_MAX_AGG_RANGES];
  /* TERMS on numeric columns: dense index = raw value; on STR: ordinal */
  uint32_t has_missing;  /* `missing` parameter present (composite: `missing_bucket`) */
  uint32_t reserved;     /* TRACE_IDS: the timestamp column; TERMS / HISTOGRAM: QW_AGG_COMP_* flags */
  uint64_t missing_value; /* mapped-u64 (numeric) or ordinal==dict_num_terms for "new key"; STATS / PERCENTILES: f64 bits */
} QwAggNode;

typedef struct QwPlanHeader {
  uint32_t magic;
  uint32_t version;
  uint32_t num_nodes; /* query nodes; node 0 is the root */
  uint32_t num_aggs;  /* QwAggNode count */
  uint32_t max_hits;  /* leaf_max_hits = max_hits + start_offset (collector.rs:772-774) */
  uint32_t scoring;   /* QuickwitCollector::requires_scoring (collector.rs:819-830) */
  uint32_t count_only; /* max_hits == 0 && no aggregation (collector.rs:723-725) */
  uint32_t reserved;   /* QW_PLAN_* flags */
  QwSortSpec sort[2];
  QwSearchAfter search_after;
  /* followed by QwPlanNode[num_nodes], then QwAggNode[num_aggs] */
} QwPlanHeader;

/* QwPlanHeader.reserved: return the hits through full QwHit records from the device even where qw_plan_score_hits()
 * holds (the results are the same; tests compare the two forms) */
#define QW_PLAN_FULL_HITS 1u

/* A hit of a plan ranked by _score descending alone, as the device hands it back: the rest of its QwHit follows
 * from these two fields (v1 = f64_to_u64(score as f64), flags = 1, v2 = reserved = 0). */
typedef struct QwScoreHit {
  uint32_t doc_id;
  float score;
} QwScoreHit;

/* 1 when the device returns the plan's hits as QwScoreHit records: sorted by _score descending with no second key
 * (a `_doc` second key extracts None), no search_after, and QW_PLAN_FULL_HITS clear. */
static inline int qw_plan_score_hits(const QwPlanHeader* h) {
  return h->sort[0].kind == QW_SORT_SCORE && h->sort[0].order == QW_ORDER_DESC &&
         (h->sort[1].kind == QW_SORT_NONE || h->sort[1].kind == QW_SORT_DOCID) && !h->search_after.present &&
         !(h->reserved & QW_PLAN_FULL_HITS);
}

/* ---------------------------------------------------------------- result --------------------- */

/* One hit of the per-split top-K, best first. v1/v2 are the u64 fast-field representations
 * (SegmentPartialHit, collector.rs:484-491); for QW_SORT_SCORE v1 = f64_to_u64(score as f64)
 * (collector.rs:180) and `score` carries the raw f32. */
typedef struct QwHit {
  uint64_t v1, v2;
  uint32_t doc_id;
  uint32_t flags; /* bit0: v1 is Some, bit1: v2 is Some */
  float score;
  uint32_t reserved;
} QwHit;

/* Dense aggregation result (plans for which qw_agg_hashed() is 0). Every QwAggNode owns `cells(node)` = Π num_buckets over its ancestor
 * chain (itself included; metric nodes count 1, a QW_AGG_STATS node with has_missing 2: its second bank, after the
 * first, holds in `count` the docs without a value per parent cell) cells, laid out row-major (outermost ancestor
 * slowest). Bucket nodes use only `count` (doc_count). Metric nodes (QW_AGG_STATS) use all four:
 * `sum_bits`: where qw_stats_sum_exact() holds, the exact integer sum of the RAW offsets (value =
 * min_value + gcd * raw in the mapped space) — the host rebuilds count * min + gcd * sum in 128-bit
 * arithmetic, so e.g. an avg over nanosecond timestamps cannot overflow; everywhere else (f64 columns,
 * wider raws, splits with too many values), the bit pattern of an f64 sum of the typed values (what
 * tantivy accumulates). min/max are in the column's mapped-u64 space (initialised to UINT64_MAX / 0).
 * The host converts to f64 when it builds the intermediate aggregation result. */
#define QW_SUM_EXACT_BITS 40u
typedef struct QwAggCell {
  uint64_t count;
  uint64_t sum_bits;
  uint64_t min_mapped;
  uint64_t max_mapped;
} QwAggCell;

/* Hashed aggregation result (DESIGN.md §4.4, hashed cells): one entry per (node, parent entry, bucket key) that
 * a matched doc of the split reached, instead of Π num_buckets dense cells per node. A split's plan takes this
 * layout when its tree is deeper than bucket -> bucket -> metric, its dense cells add up to more than
 * QW_AGG_DENSE_MAX_CELLS, or a TERMS node's dense space exceeds QW_AGG_DENSE_MAX_TERMS (qw_agg_hashed).
 *   key: TERMS = the bit-packed raw value (0 with QW_AGG_ENTRY_MISSING: the `missing` bucket); HISTOGRAM = the
 *        bucket index relative to base_pos (agg_bucket's f64 formula); RANGE = the range index; STATS = 0 (with
 *        QW_AGG_ENTRY_MISSING: the count of docs without a value);
 *        PERCENTILES = the index of the value's bin in the split's boundary table (QW_AGG_PERCENTILES).
 *   cell: as in the dense layout (bucket entries use `count` only). */
#define QW_AGG_DENSE_MAX_CELLS (1ull << 26)
#define QW_AGG_DENSE_MAX_TERMS (1ull << 24)
#define QW_AGG_NO_PARENT 0xFFFFFFFFu
enum { QW_AGG_ENTRY_MISSING = 1u };
typedef struct QwAggEntry {
  uint32_t node;
  uint32_t parent; /* index of the parent bucket's entry; QW_AGG_NO_PARENT for top-level nodes */
  uint64_t key;
  uint32_t flags;  /* QW_AGG_ENTRY_* */
  uint32_t reserved;
  QwAggCell cell;
} QwAggEntry; /* 56 bytes */

/* 1 when the plan's aggregation tree takes the hashed layout: a composite source node, a percentiles node, a node below two bucket ancestors that is not a
 * metric (or any node below three), the dense cells of all nodes adding up to more than QW_AGG_DENSE_MAX_CELLS,
 * or a TERMS node whose dense space (num_buckets without the `missing` slot) exceeds QW_AGG_DENSE_MAX_TERMS.
 * Reads only the plan; the caller has checked every parent index. */
static inline int qw_agg_hashed(const QwAggNode* nodes, uint32_t n) {
  uint64_t total = 0;
  for (uint32_t i = 0; i < n; i++) {
    const QwAggNode* g = &nodes[i];
    if ((g->kind == QW_AGG_TERMS || g->kind == QW_AGG_HISTOGRAM) && (g->reserved & QW_AGG_COMP_LEVEL)) return 1;
    if (g->kind == QW_AGG_PERCENTILES) return 1;
    if (g->kind == QW_AGG_TERMS && (uint64_t)g->num_buckets - (g->has_missing ? 1u : 0u) > QW_AGG_DENSE_MAX_TERMS) return 1;
    uint32_t depth = 0;
    uint64_t cells = g->kind == QW_AGG_STATS ? (g->has_missing ? 2 : 1) : g->num_buckets;
    for (uint32_t p = g->parent; p != 0xFFFFFFFFu; p = nodes[p].parent) {
      depth++;
      if (depth > n) return 1; /* (a parent cycle: lowering refuses it) */
      cells *= nodes[p].num_buckets;
      if (cells > QW_AGG_DENSE_MAX_CELLS) cells = QW_AGG_DENSE_MAX_CELLS + 1;
    }
    if (depth > 2 || (depth == 2 && g->kind != QW_AGG_STATS)) return 1;
    total += cells;
    if (total > QW_AGG_DENSE_MAX_CELLS) return 1;
  }
  return 0;
}

static inline uint32_t qw_bit_length(uint64_t x) {
  uint32_t n = 0;
  while (x) { n++; x >>= 1; }
  return n;
}
/* How stats node `ni` sums its column in one split (the GPU engine, the host finalisation and the CPU oracle
 * all decide here): 1 = the exact u64 sum of raw offsets, 0 = an f64 sum. The exact sum is only chosen when it
 * cannot wrap: an integer-typed column with raws of at most QW_SUM_EXACT_BITS bits, and fewer than
 * 2^(64 - bits) raws added into any one cell. A cell adds each value of the column at most once per value of a
 * multi-valued ancestor bucket column that put the doc in it, so those columns' value counts bound the total
 * too. A split of 2^24 docs with six nanosecond timestamps each (40 bits) would wrap without this rule. */
static inline int qw_stats_sum_exact(const QwImgColumn* cols, const QwAggNode* nodes, uint32_t ni) {
  const QwAggNode* g = &nodes[ni];
  if (g->column == 0xFFFFFFFFu) return 0;
  const QwImgColumn* c = &cols[g->column];
  if (c->type == QW_COL_F64 || c->bits > QW_SUM_EXACT_BITS) return 0;
  uint32_t width = c->bits + qw_bit_length(c->num_vals);
  for (uint32_t p = g->parent; p != 0xFFFFFFFFu; p = nodes[p].parent)
    if (nodes[p].column != 0xFFFFFFFFu && cols[nodes[p].column].cardinality == QW_CARD_MULTI)
      width += qw_bit_length(cols[nodes[p].column].num_vals);
  return width <= 64;
}

#ifdef __cplusplus
}
#endif
#endif /* QWGPU_FORMAT_H */
