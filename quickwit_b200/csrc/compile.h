// compile.h — host-side request compilation + aggregation result plumbing (declarations).
#pragma once
#include <optional>
#include <string>
#include <vector>

#include "common.h"
#include "json.h"
#include "proto.h"

namespace qw {

// The subset of Quickwit's doc mapper JSON this path needs
// (quickwit-doc-mapper/src/doc_mapper/{doc_mapper_builder.rs,field_mapping_entry.rs}).
struct DocMapperInfo {
  struct Field { std::string name, type, tokenizer, fast_precision; };
  std::string timestamp_field;
  std::vector<Field> fields;
  std::vector<std::string> default_search_fields;
};
DocMapperInfo parse_doc_mapper(const std::string& json);
std::vector<std::string> tokenize_text(const std::string& text, uint32_t tokenizer);
bool parse_datetime_str(const std::string& s, int64_t* nanos);

// ---- aggregation request (tantivy::aggregation::agg_req::Aggregations, Elasticsearch-shaped JSON;
// semantics per docs/reference/aggregation.md) --------------------------------------------------------
struct AggReq {
  // TraceIds: quickwit's FindTraceIdsCollector (find_trace_ids_collector.rs), which takes the place of the whole
  // aggregation request (`size` = num_traces, `field` = trace_id_field_name, `ts_field` = span_timestamp_field_name)
  enum Kind { Terms, Histogram, DateHistogram, Range, Stats, Avg, Sum, Min, Max, Count, TraceIds } kind = Terms;
  std::string ts_field;
  uint64_t num_traces = 0;
  std::string name, field;
  // terms
  uint32_t size = 10, segment_size = 100;
  uint64_t min_doc_count = 1;  // terms default 1, histogram default 0
  bool has_missing = false;
  Json missing;
  std::string order_target = "_count";
  bool order_desc = true;
  // histogram / date_histogram (interval and offset in REQUEST units: ms for date_histogram)
  double interval = 0, offset = 0;
  bool has_hard_bounds = false, has_extended_bounds = false, keyed = false;
  double hard_min = 0, hard_max = 0, ext_min = 0, ext_max = 0;
  // range
  struct R { bool has_from = false, has_to = false; double from = 0, to = 0; std::string key; };
  std::vector<R> ranges;
  std::vector<AggReq> children;
  bool is_metric() const { return kind >= Stats && kind <= Count; }
};
std::vector<AggReq> parse_agg_request(const std::string& json);
inline bool is_trace_ids_request(const std::vector<AggReq>& r) { return r.size() == 1 && r[0].kind == AggReq::TraceIds; }

// find_trace_ids results: Vec<Span> in postcard (varint length; per span the 16 trace-id bytes and the zigzag varint
// of the i64 timestamp in ns), the bytes the reference puts into intermediate_aggregation_result
struct TraceSpan {
  uint8_t id[16];
  int64_t ts;
};
bool span_less(const TraceSpan& a, const TraceSpan& b);  // Span::cmp: timestamp desc, then trace id bytes asc
std::string encode_spans(const std::vector<TraceSpan>& v);
std::vector<TraceSpan> decode_spans(const std::string& bytes);
// merge_segment_fruits: sort each fruit, k-merge, keep the first span of every trace id, stop at num_traces
std::vector<TraceSpan> merge_span_fruits(std::vector<std::vector<TraceSpan>> fruits, uint64_t num_traces);

// How one QwAggNode of a split maps dense bucket indices back to keys
struct AggBinding {
  const AggReq* req = nullptr;
  int column = -1;
  uint32_t col_type = 0;
};
// Flattens the request against one split (column lookup, dense bucket space); nodes are emitted
// breadth-first so that the children of a node are contiguous.
std::vector<QwAggNode> lower_aggs(const std::vector<AggReq>& reqs, const ImageView& img, std::vector<AggBinding>& bindings);

struct CompiledPlan {
  std::string bytes;  // QwPlanHeader + nodes + agg nodes
  QwPlanHeader header;
  int sort_field_type[2] = {0, 0};
  std::vector<AggReq> agg_request;
  std::vector<AggBinding> agg_bindings;  // parallel to the plan's QwAggNode[]; point into agg_request
};
// `parsed_ast`: the request's query_ast already parsed (one parse per leaf request, not per split)
CompiledPlan compile_plan(const ImageView& img, const std::string& split_id, const pb::SearchRequest& req,
                          const DocMapperInfo& dm, const pb::SplitIdAndFooterOffsets* split_meta,
                          const Json* parsed_ast = nullptr);

// ---- intermediate aggregation results (role of tantivy's IntermediateAggregationResults; our own
// postcard-style byte layout — the reference layout is a tantivy-internal struct, SURVEY.md §7 hard
// part iv) -----------------------------------------------------------------------------------------------
std::string build_intermediate_aggs(const CompiledPlan& cp, const ImageView& img, const QwAggCell* cells, size_t ncells);
std::string merge_intermediate_aggs(const std::vector<AggReq>& reqs, const std::vector<std::string>& parts);
struct SplitAggCells {
  const CompiledPlan* plan;
  const ImageView* img;
  const QwAggCell* cells;
  size_t ncells;
};
std::string build_and_merge_intermediate_aggs(const std::vector<AggReq>& reqs, const std::vector<SplitAggCells>& splits);
std::string finalize_aggs_json(const std::vector<AggReq>& reqs, const std::string& intermediate);

// ---- per-split response + merging ---------------------------------------------------------------------
// SegmentPartialHit::into_partial_hit (collector.rs:493-521): QwHit -> PartialHit with typed sort values
pb::LeafSearchResponse build_split_response(const CompiledPlan& cp, const ImageView& img, const std::string& split_id,
                                            uint64_t num_hits, const QwHit* hits, size_t nhits,
                                            const QwAggCell* cells, size_t ncells);
// merge_leaf_responses + merge_fruits truncation (collector.rs:832-974)
pb::LeafSearchResponse merge_responses(const pb::SearchRequest& req, std::vector<pb::LeafSearchResponse> parts);

}  // namespace qw
