/*
 * qwgpu.h — C ABI of libqwgpu.so: the H100-native drop-in for Quickwit's per-split leaf search.
 *
 * What each entry point replaces in the reference (paths relative to
 * the quickwit-oss/quickwit repository @ 544b50f):
 *
 *   qwgpu_leaf_search          SearchService::leaf_search(LeafSearchRequest) -> LeafSearchResponse
 *                              quickwit-search/src/service.rs:81,177-203 (seam A, SURVEY.md §3.4)
 *   qwgpu_invoke_leaf_search   LambdaLeafSearchInvoker::invoke_leaf_search(LeafSearchRequest)
 *                              -> Vec<LambdaSingleSplitResult>; quickwit-search/src/invoker.rs:27-38
 *                              (seam B; response = LambdaSearchResponses-shaped bytes)
 *   qwgpu_split_search         searcher.search(&query, &collector) for ONE split,
 *                              quickwit-search/src/leaf.rs:637 (seam C; plan in, hits/buckets out)
 *   qwgpu_compile_plan         doc_mapper.query(...) + make_collector_for_split(...):
 *                              quickwit-search/src/leaf.rs:562-580, collector.rs:1033-1052,
 *                              quickwit-query/src/query_ast/tantivy_query_ast.rs:166-377
 *   qwgpu_merge_leaf_responses QuickwitCollector::merge_fruits / merge_leaf_responses /
 *                              IncrementalCollector, quickwit-search/src/collector.rs:832-974,1195-1313
 *                              (leaf-level and root-level merge; called from root.rs:836-853)
 *   qwgpu_finalize_aggregation finalize_aggregation, quickwit-search/src/root.rs:1105-1135
 *   qwgpu_split_register       open_index_with_caches + warmup (leaf.rs:210-251,269-472): makes
 *                              a split's postings / columns / fieldnorms resident — in HBM.
 *   qwgpu_imgb_*               the split-image writer (the transcoding target for a tantivy
 *                              segment; SURVEY.md §8f-2). Not on the query path.
 *
 * Conventions: every function returns 0 on success, a negative QWGPU_E* code otherwise;
 * qwgpu_last_error() returns a thread-local message (maps to SearchError::Internal /
 * InvalidQuery / InvalidAggregationRequest / InvalidArgument, quickwit-search/src/error.rs:32-53).
 * Buffers returned through `uint8_t** out` are malloc'ed by the library and released with
 * qwgpu_buf_free. All entry points are thread-safe and re-entrant on a ctx
 * (the reference calls leaf search concurrently from its rayon pool, SURVEY.md §8b "Threading").
 * There is NO CPU fallback: search entry points fail with QWGPU_ENODEVICE without a CUDA device.
 */
#ifndef QWGPU_H
#define QWGPU_H

#include <stddef.h>
#include <stdint.h>

#include "qwgpu_format.h"

#ifdef __cplusplus
extern "C" {
#endif

#define QWGPU_OK 0
#define QWGPU_EINTERNAL (-1)      /* SearchError::Internal */
#define QWGPU_EINVALID_QUERY (-2) /* SearchError::InvalidQuery */
#define QWGPU_EINVALID_AGG (-3)   /* SearchError::InvalidAggregationRequest */
#define QWGPU_EINVALID_ARG (-4)   /* SearchError::InvalidArgument */
#define QWGPU_ENODEVICE (-5)      /* no CUDA device: the product path never falls back to CPU */
#define QWGPU_ENOTFOUND (-6)      /* unknown split id */
#define QWGPU_EUNSUPPORTED (-7)   /* query/aggregation shape not implemented on the GPU path */

typedef struct qwgpu_ctx qwgpu_ctx;
typedef struct qwgpu_imgb qwgpu_imgb;

const char* qwgpu_last_error(void);
const char* qwgpu_version(void);
void qwgpu_buf_free(void* buf);

/* ---- context ------------------------------------------------------------------------------- */

/* device < 0: host-only context (plan compilation, merging; no search). */
int qwgpu_init(int device, qwgpu_ctx** out);
void qwgpu_shutdown(qwgpu_ctx* ctx);

/* Copies the image's data region to the device; the host-side directory (term dictionary,
 * column dictionaries, headers) is copied and owned by the ctx. `img` may be freed afterwards. */
int qwgpu_split_register(qwgpu_ctx* ctx, const char* split_id, const uint8_t* img, uint64_t img_len);
int qwgpu_split_unregister(qwgpu_ctx* ctx, const char* split_id);
/* Bytes resident on the device for this ctx. */
uint64_t qwgpu_resident_bytes(qwgpu_ctx* ctx);

/* Residency manager — the GPU-side counterpart of a searcher's split cache and of the open + warmup step of a
 * leaf search (quickwit-search/src/leaf.rs:210-251 open_split_bundle, :269-472 warmup):
 *   qwgpu_set_residency_budget  cap on the bytes of split data kept in HBM (0 = none). A registration that does
 *                               not fit evicts the least recently searched splits that no running call uses; a
 *                               search on an evicted split reports it in failed_splits (retryable: the caller
 *                               registers it again), exactly like a split that was never registered.
 *   qwgpu_split_register_async  returns at once; the data region is uploaded by a background thread through
 *                               pinned staging buffers on its own stream, searches on other splits keep running.
 *                               `img` must stay valid until qwgpu_split_wait(split_id) has returned. A search
 *                               that names a split still loading waits for it.
 *   qwgpu_split_wait            blocks until the upload has finished; returns its error, if any.
 *   qwgpu_residency_info        bytes resident, budget, number of splits, evictions so far (NULL = not wanted). */
int qwgpu_set_residency_budget(qwgpu_ctx* ctx, uint64_t bytes);
int qwgpu_split_register_async(qwgpu_ctx* ctx, const char* split_id, const uint8_t* img, uint64_t img_len);
int qwgpu_split_wait(qwgpu_ctx* ctx, const char* split_id);
int qwgpu_residency_info(qwgpu_ctx* ctx, uint64_t* resident_bytes, uint64_t* budget_bytes, uint64_t* num_splits, uint64_t* evictions);
int qwgpu_split_is_resident(qwgpu_ctx* ctx, const char* split_id);

/* ---- seam A / B: protobuf in, protobuf out ---------------------------------------------------- */

/* req = quickwit.search.LeafSearchRequest, resp = quickwit.search.LeafSearchResponse
 * (quickwit-proto/protos/quickwit/search.proto:343-359,583-613). Per-split failures are reported
 * in `failed_splits` (retryable_error = true), never as a non-zero return (leaf.rs:1989-2004). */
int qwgpu_leaf_search(qwgpu_ctx* ctx, const uint8_t* req, size_t req_len, uint8_t** resp,
                      size_t* resp_len);
/* resp = quickwit.search.LambdaSearchResponses (one LambdaSingleSplitResult per split). */
int qwgpu_invoke_leaf_search(qwgpu_ctx* ctx, const uint8_t* req, size_t req_len, uint8_t** resp,
                             size_t* resp_len);

/* ---- seam C: plan in, hits / buckets out ------------------------------------------------------- */

/* Compiles (SearchRequest protobuf, doc mapper JSON) against ONE split image into a QwPlanHeader
 * blob (host only; works on a device-less ctx). `img` is any registered-or-not split image. */
int qwgpu_compile_plan(const uint8_t* img, uint64_t img_len, const char* split_id,
                       const uint8_t* search_request_pb, size_t search_request_len,
                       const char* doc_mapper_json, uint8_t** plan, size_t* plan_len);

typedef struct qwgpu_split_result {
  uint64_t num_hits;
  uint32_t num_partial_hits; /* <= plan.max_hits */
  uint32_t num_agg_cells;    /* total cells over all QwAggNode, node-major */
  QwHit* hits;               /* malloc'ed; free with qwgpu_buf_free */
  QwAggCell* agg_cells;      /* malloc'ed; free with qwgpu_buf_free */
  /* measurement: device time of the search kernels of this call (CUDA events), microseconds */
  float gpu_time_us;
  float main_kernel_us;      /* device time of the dominant kernel (k_window<COLLECT>) of this call */
  uint32_t num_kernel_launches;
  uint32_t exact_fallbacks;  /* 1 when the sampled top-K threshold failed verification */
  uint64_t postings_scored; /* Σ doc_freq of the plan's terms ("docs scored", SURVEY.md §8d) */
  uint64_t algorithmic_bytes; /* SURVEY.md §8d numerator for this split/plan */
  /* The path the call took (DESIGN.md §4.6). Per call: every split of the batch reports the same values. */
  uint32_t kernel_mask;      /* QWGPU_KERNEL_* bits of the search kernels launched */
  uint32_t window_docs;      /* docs per work item: the window size W, the driving term's block size (128) for
                                k_driver, the 8192-doc chunk for k_aggscan */
  uint32_t sample_stride;    /* stride of the sampled top-K threshold pass; 0 when no sampled pass ran */
  uint32_t radix_passes;     /* exact radix rounds (histogram pass + digit pick) of the top-K threshold */
  uint32_t refined;          /* 1 when a failed sampled threshold was repaired by the candidates-only pass */
} qwgpu_split_result;

/* qwgpu_split_result.kernel_mask */
#define QWGPU_KERNEL_UNION 1u   /* k_union: BM25 unions (TMA + mbarrier pipeline) */
#define QWGPU_KERNEL_DRIVER 2u  /* k_driver: one driving posting list + column filters */
#define QWGPU_KERNEL_AGGSCAN 4u /* k_aggscan: match_all + flat aggregations */
#define QWGPU_KERNEL_WINDOW 8u  /* k_window: the generic window kernel */
#define QWGPU_KERNEL_PHRASE 16u /* k_phrase: the phrase pre-pass */
#define QWGPU_KERNEL_TRACE_SELECT 32u /* k_trace_select: find_trace_ids top N over the per-trace maxima */
#define QWGPU_KERNEL_TRACE_REPLAY 64u /* k_trace_replay: the reference's sentinel replay on a split whose N-th and
                                         (N+1)-th trace timestamps tie */

/* Runs `num_splits` plans (plan i against split_ids[i]) in ONE batched launch sequence.
 * results[i] is filled for every split; status[i] is 0 or a QWGPU_E* code for that split. */
int qwgpu_split_search(qwgpu_ctx* ctx, uint32_t num_splits, const char* const* split_ids,
                       const uint8_t* const* plans, const size_t* plan_lens,
                       qwgpu_split_result* results, int* status);
void qwgpu_split_result_free(qwgpu_split_result* r);

/* Builds the per-split LeafSearchResponse protobuf (typed sort values, intermediate aggregation
 * bytes) from a seam-C result: QuickwitSegmentCollector::harvest, collector.rs:564-594. Host only. */
int qwgpu_build_leaf_response(const uint8_t* img, uint64_t img_len, const char* split_id,
                              const uint8_t* search_request_pb, size_t search_request_len,
                              const char* doc_mapper_json, uint64_t num_hits, const QwHit* hits,
                              uint32_t num_partial_hits, const QwAggCell* cells, uint32_t num_cells,
                              uint8_t** resp, size_t* resp_len);

/* Pre-search pruning (SURVEY.md 8a row a16), host only: what qwgpu_leaf_search does to the request of every
 * split before it searches — CanSplitDoBetter::{from_request, optimize_split_order, optimize}
 * (quickwit-search/src/leaf.rs:1072-1242), disable_search_request_hits (leaf.rs:1438-1443) and
 * is_metadata_count_request_with_ast (root.rs:665-686; leaf.rs:525-528 answers such a split from num_docs) and
 * simplify_search_request (leaf.rs:1399-1433: under CountHits::Underestimate a split that has neither hits nor an
 * aggregation left to compute is not searched at all — "skipped").
 * `json_out` (qwgpu_buf_free) = [{"split_id", "max_hits", "hits_disabled", "metadata_count", "skipped"}, ...] in the
 * reference's processing order, one entry per split of the request. */
int qwgpu_optimize_leaf_request(const uint8_t* leaf_search_request_pb, size_t req_len, uint8_t** json_out, size_t* json_len);

/* ---- merge / finalize -------------------------------------------------------------------------- */

/* Merges N LeafSearchResponse protobufs under `search_request_pb` (sort orders, max_hits,
 * start_offset, aggregation request): semantics of merge_leaf_responses +
 * QuickwitCollector::merge_fruits (collector.rs:832-974). */
int qwgpu_merge_leaf_responses(const uint8_t* search_request_pb, size_t search_request_len,
                               uint32_t n, const uint8_t* const* resps, const size_t* resp_lens,
                               uint8_t** merged, size_t* merged_len);
/* intermediate aggregation bytes -> final aggregation JSON (root.rs:1105-1135). */
int qwgpu_finalize_aggregation(const char* aggregation_request_json, const uint8_t* intermediate,
                               size_t intermediate_len, char** json_out);

/* ---- multi-GPU partial exchange (SURVEY.md §8e) -------------------------------------------------
 * Fixed-layout per-rank partial: what one rank contributes to the single all-gather that stands in
 * for the root merge — counters, up to max_hits + start_offset typed hits, a bounded tail holding the
 * failed_splits entries and resource statistics, and the intermediate aggregation bytes. The caller (one process per GPU) all-gathers `partial_bytes` from every
 * rank (NCCL) and calls qwgpu_merge_partials on the gathered buffer (every rank or rank 0). */
int qwgpu_partial_size(const uint8_t* search_request_pb, size_t search_request_len,
                       uint64_t* partial_bytes);
int qwgpu_response_to_partial(const uint8_t* search_request_pb, size_t search_request_len,
                              const uint8_t* resp, size_t resp_len, uint8_t* partial,
                              uint64_t partial_bytes);
int qwgpu_merge_partials(const uint8_t* search_request_pb, size_t search_request_len,
                         uint32_t n_ranks, const uint8_t* gathered, uint64_t partial_bytes,
                         uint8_t** merged, size_t* merged_len);

/* Device-side exchange (one process per GPU, NCCL over NVLink): the all-gather that stands in for the root
 * merge (quickwit-search/src/root.rs:836-853 -> collector.rs:914-974) runs inside the library, on the
 * call's stream, on device-resident records, and the gathered lists are merged on the device.
 *   qwgpu_comm_unique_id       rank 0 creates the 128-byte NCCL id and hands it to the other ranks
 *   qwgpu_comm_init            every rank: builds the communicator for this context's device
 *   qwgpu_comm_set_split_table every rank: the split ids of the whole (multi-GPU) index, any order; their
 *                              sorted position is the tie-break rank carried by the exchanged hits
 *   qwgpu_leaf_search_allgather  collective: leaf_search on this rank's splits + exchange; every rank gets
 *                              the merged LeafSearchResponse. Top-K requests without aggregations take the
 *                              device road (record = counters + best k hits, one ncclAllGather on the call's
 *                              stream, device merge). Requests with aggregations or without hits, and any
 *                              request for which some rank reports a failed split, take the host-staged
 *                              road: each rank's complete response as a fixed-layout partial (hits,
 *                              aggregation bytes, failed_splits entries, resource statistics), only its used
 *                              prefix on the wire (two ncclAllGather calls: lengths, then payload), merged
 *                              with qwgpu_merge_partials' code on every rank. A rank whose own search fails
 *                              still takes part and reports its splits as failed (retryable). */
int qwgpu_comm_unique_id(uint8_t* out128);
int qwgpu_comm_init(qwgpu_ctx* ctx, const uint8_t* id128, int rank, int world);
int qwgpu_comm_set_split_table(qwgpu_ctx* ctx, uint32_t n, const char* const* split_ids);
void qwgpu_comm_destroy(qwgpu_ctx* ctx);
int qwgpu_leaf_search_allgather(qwgpu_ctx* ctx, const uint8_t* leaf_search_request_pb, size_t len,
                                uint8_t** merged_resp, size_t* merged_len);
/* Lanes: the collectives of one NCCL communicator must be issued in the same order on every rank, so one
 * communicator serialises the searches that use it. A context holds up to 16 communicators ("lanes", each with
 * its own unique id; lane 0 = qwgpu_comm_init): concurrent searches — one host thread per lane, the same
 * assignment of requests to lanes on every rank — overlap like concurrent qwgpu_leaf_search calls do. */
int qwgpu_comm_init_lane(qwgpu_ctx* ctx, uint32_t lane, const uint8_t* id128, int rank, int world);
int qwgpu_leaf_search_allgather_lane(qwgpu_ctx* ctx, uint32_t lane, const uint8_t* leaf_search_request_pb, size_t len,
                                     uint8_t** merged_resp, size_t* merged_len);

/* ---- real `.split` files ------------------------------------------------------------------------
 * Reads the footer of a Quickwit split bundle: `tail` = the last `tail_len` bytes of the split file (at least
 * [split_footer_start, split_footer_end) of SplitIdAndFooterOffsets, search.proto:489-503), `split_file_len` =
 * the size of the whole file. Layout (quickwit-storage/src/bundle_storage.rs:92-174,
 * quickwit-directories/src/hot_directory.rs:40-80): ...files | BundleStorageFileOffsets (versioned header + JSON)
 * | u32 len | hotcache (versioned header + postcard HotDirectoryMeta + cached slices) | u32 len.
 * `json_out` (qwgpu_buf_free): {"files": [{"path", "start", "end"}] sorted by offset, "bundle_metadata": {"offset",
 * "len"}, "footer_start", "footer_end", "hotcache": {"offset", "len", "file_lengths": {path: len}, "slices":
 * [{"path", "offset"}]}} — every offset is a byte offset in the split file. Host only; the first step of ingesting
 * a real split (SURVEY.md 8f-2): it locates the tantivy .term / .idx / .pos / .fast / .fieldnorm files. */
int qwgpu_parse_split_footer(const uint8_t* tail, uint64_t tail_len, uint64_t split_file_len, uint8_t** json_out, size_t* json_len);

/* ---- split image writer ------------------------------------------------------------------------ */

qwgpu_imgb* qwgpu_imgb_new(uint32_t num_docs);
void qwgpu_imgb_free(qwgpu_imgb* b);
/* returns field id (>= 0) or a negative error. fieldnorm_ids: num_docs bytes or NULL. */
int qwgpu_imgb_add_field(qwgpu_imgb* b, const char* name, uint32_t flags, uint32_t tokenizer,
                         const uint8_t* fieldnorm_ids, uint64_t total_num_tokens);
/* docs strictly increasing; tfs NULL when the field has no freqs. */
int qwgpu_imgb_add_term(qwgpu_imgb* b, uint32_t field_id, const uint8_t* term, uint32_t term_len,
                        const uint32_t* docs, const uint32_t* tfs, uint32_t n);
/* Fields with QW_FIELD_HAS_POSITIONS (`record: position`): the same plus the token positions of every posting —
 * tfs[i] strictly increasing positions per posting, concatenated in posting order (n_positions = sum of tfs). */
int qwgpu_imgb_add_term_positions(qwgpu_imgb* b, uint32_t field_id, const uint8_t* term, uint32_t term_len,
                                  const uint32_t* docs, const uint32_t* tfs, uint32_t n,
                                  const uint32_t* positions, uint64_t n_positions);
/* values: mapped-u64 values. index: FULL -> NULL (num_vals == num_docs);
 * OPTIONAL -> sorted doc ids (num_vals of them); MULTI -> start offsets (num_docs + 1).
 * STR columns pass ordinals as values plus the sorted dictionary. */
int qwgpu_imgb_add_column(qwgpu_imgb* b, const char* name, uint32_t type, uint32_t cardinality,
                          const uint64_t* values, uint64_t num_vals, const uint32_t* index,
                          const uint8_t* dict_bytes, const uint32_t* dict_offs, uint32_t dict_n);
int qwgpu_imgb_finish(qwgpu_imgb* b, uint8_t** img, uint64_t* img_len);

/* Synthetic hdfs-logs-shaped split (SURVEY.md §8d corpus): see DESIGN.md "Synthetic corpus".
 * term_fracs[i] is the doc-frequency fraction of body term "t<i>"; deterministic in `seed`. */
typedef struct qwgpu_synth_spec {
  uint32_t num_docs;
  uint32_t split_ord;
  uint64_t seed;
  uint32_t num_terms;
  const double* term_fracs;
  int64_t ts_start_secs; /* first timestamp; docs advance monotonically, 1 s resolution */
  uint32_t ts_span_secs; /* timestamps cover [ts_start, ts_start + span) */
  uint32_t num_tenants;
  /* > 0: a second text field "msg", indexed with positions (`record: position`): 4..8 tokens per doc drawn
   * Zipf(1) from the vocabulary "w0".."w<msg_vocab-1>" — the field the phrase queries of BASELINE config 5 run on */
  uint32_t msg_vocab;
  uint32_t reserved;
} qwgpu_synth_spec;
int qwgpu_synth_split(const qwgpu_synth_spec* spec, uint8_t** img, uint64_t* img_len);

/* Bm25Weight of one term: idf(doc_freq, num_docs) * (1 + K1) * boost in f32 (what
 * qwgpu_compile_plan writes into QwPlanNode.bm25_weight); for hand-built seam-C plans. */
float qwgpu_bm25_weight(uint64_t doc_freq, uint64_t num_docs, float boost);
/* PhraseWeight's Bm25Weight::for_terms: (sum of the terms' idf in phrase order, f32) * (1 + K1) * boost. */
float qwgpu_bm25_phrase_weight(const uint64_t* doc_freqs, uint32_t n, uint64_t num_docs, float boost);

/* tantivy fieldnorm <-> id table (tantivy::fieldnorm::{fieldnorm_to_id,id_to_fieldnorm}). */
uint8_t qwgpu_fieldnorm_to_id(uint32_t fieldnorm);
uint32_t qwgpu_id_to_fieldnorm(uint8_t id);

#ifdef __cplusplus
}
#endif
#endif /* QWGPU_H */
