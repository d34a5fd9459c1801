// leaf.cpp — the leaf-search surface on top of the GPU engine:
//   * build_split_response    QuickwitSegmentCollector::harvest + SegmentPartialHit::into_partial_hit
//                             (quickwit-search/src/collector.rs:493-521,564-594)
//   * merge_responses         merge_leaf_responses / merge_fruits / IncrementalCollector
//                             (collector.rs:832-992,1195-1313), SortValue total order
//                             (quickwit-proto/src/search/mod.rs:137-161), add_leaf_stats (lib.rs:392-425)
//   * qwgpu_leaf_search       SearchService::leaf_search -> multi_index_leaf_search ->
//                             single_doc_mapping_leaf_search (service.rs:177-203, leaf.rs:1290-1394,1673-1791)
//   * qwgpu_invoke_leaf_search LambdaLeafSearchInvoker::invoke_leaf_search (invoker.rs:27-38;
//                             handler template quickwit-lambda-server/src/handler.rs:55-200)
//   * partial exchange for the multi-GPU root merge stand-in (SURVEY.md §8e)
//   * LeafCache               LeafSearchCache (quickwit-search/src/leaf_cache.rs:27-185), read and written like
//                             leaf.rs:510-517,695-705,1872-1896
#include <algorithm>
#include <chrono>
#include <tuple>

#include "regex.h"
#include "compile.h"
#include "ddsketch.h"
#include "device_types.h"
#include "engine.h"
#include "comm.h"

namespace qw {

// ---- SortValue order (quickwit-proto/src/search/mod.rs:137-161) ----------------------------------------
static int cmp_i(int64_t a, int64_t b) { return a < b ? -1 : (a > b ? 1 : 0); }
static int cmp_u(uint64_t a, uint64_t b) { return a < b ? -1 : (a > b ? 1 : 0); }
static int total_cmp(double a, double b) {  // f64::total_cmp
  int64_t x, y;
  memcpy(&x, &a, 8);
  memcpy(&y, &b, 8);
  x ^= (int64_t)((uint64_t)(x >> 63) >> 1);
  y ^= (int64_t)((uint64_t)(y >> 63) >> 1);
  return cmp_i(x, y);
}
static int sortvalue_cmp(const pb::SortValue& a, const pb::SortValue& b) {
  using SV = pb::SortValue;
  if (a.kind == SV::U64 && b.kind == SV::U64) return cmp_u(a.u, b.u);
  if (a.kind == SV::I64 && b.kind == SV::I64) return cmp_i(a.i, b.i);
  if (a.kind == SV::Bool && b.kind == SV::Bool) return cmp_i(a.b, b.b);
  if (a.kind == SV::U64 && b.kind == SV::I64) { if (a.u > (uint64_t)INT64_MAX) return 1; return cmp_i((int64_t)a.u, b.i); }
  if (a.kind == SV::F64 && b.kind == SV::F64) return total_cmp(a.f, b.f);
  if (a.kind == SV::F64 && b.kind == SV::U64) return total_cmp(a.f, (double)b.u);
  if (a.kind == SV::F64 && b.kind == SV::I64) return total_cmp(a.f, (double)b.i);
  if (a.kind == SV::Bool) { SV l; l.kind = SV::U64; l.u = a.b; return sortvalue_cmp(l, b); }
  return -sortvalue_cmp(b, a);
}
static int order_cmp_opt_sv(int order, const pb::SortValue* a, const pb::SortValue* b) {
  if (a && b) { int c = sortvalue_cmp(*a, *b); return order == QW_ORDER_DESC ? c : -c; }
  if (a) return 1;
  if (b) return -1;
  return 0;
}
// PartialHitSortingKey::cmp (collector.rs:1130-1153); > 0 when a is better
static int hit_cmp(int order1, int order2, const pb::PartialHit& a, const pb::PartialHit& b) {
  auto sv = [](bool has, const pb::SortValue& v) { return has && v.kind != pb::SortValue::None ? &v : nullptr; };
  int c = order_cmp_opt_sv(order1, sv(a.has_sv1, a.sv1), sv(b.has_sv1, b.sv1));
  if (c) return c;
  c = order_cmp_opt_sv(order2, sv(a.has_sv2, a.sv2), sv(b.has_sv2, b.sv2));
  if (c) return c;
  // GlobalDocAddress (split, segment_ord, doc_id), quickwit-search/src/lib.rs:107-131
  int d = a.split_id.compare(b.split_id);
  d = d < 0 ? -1 : (d > 0 ? 1 : 0);
  if (!d) d = cmp_u(a.segment_ord, b.segment_ord);
  if (!d) d = cmp_u(a.doc_id, b.doc_id);
  return order1 == QW_ORDER_DESC ? d : -d;
}

static void sort_orders(const pb::SearchRequest& req, int* o1, int* o2) {
  // sort_by_from_request + SortByPair::sort_orders (collector.rs:66-76,994-1030)
  *o1 = QW_ORDER_DESC;
  *o2 = QW_ORDER_DESC;
  if (req.sort_fields.size() >= 1) *o1 = req.sort_fields[0].sort_order == 0 ? QW_ORDER_ASC : QW_ORDER_DESC;
  if (req.sort_fields.size() >= 2) *o2 = req.sort_fields[1].sort_order == 0 ? QW_ORDER_ASC : QW_ORDER_DESC;
}

// convert_u64_ff_val_to_sort_value (collector.rs:183-205)
static pb::SortValue typed_sort_value(uint32_t kind, int sft, uint64_t v) {
  pb::SortValue s;
  if (kind == QW_SORT_SCORE) { s.kind = pb::SortValue::F64; s.f = u64_to_f64(v); return s; }
  if (kind == QW_SORT_DOCID) { s.kind = pb::SortValue::U64; s.u = v; return s; }
  switch (sft) {
    case 0: s.kind = pb::SortValue::U64; s.u = v; break;
    case 1: case 3: s.kind = pb::SortValue::I64; s.i = u64_to_i64(v); break;
    case 2: s.kind = pb::SortValue::F64; s.f = u64_to_f64(v); break;
    default: s.kind = pb::SortValue::Bool; s.b = v != 0; break;
  }
  return s;
}

pb::LeafSearchResponse build_split_response(const CompiledPlan& cp, const ImageView& img, const std::string& split_id,
                                            uint64_t num_hits, const QwHit* hits, size_t nhits,
                                            const QwAggCell* cells, size_t ncells,
                                            const QwAggEntry* entries, size_t nentries, bool hashed) {
  pb::LeafSearchResponse r;
  r.num_hits = num_hits;
  r.num_attempted_splits = 1;
  r.num_successful_splits = 1;
  for (size_t i = 0; i < nhits; i++) {
    pb::PartialHit h;
    h.split_id = split_id;
    h.segment_ord = 0;
    h.doc_id = hits[i].doc_id;
    if (hits[i].flags & 1) { h.has_sv1 = true; h.sv1 = typed_sort_value(cp.header.sort[0].kind, cp.sort_field_type[0], hits[i].v1); }
    if (hits[i].flags & 2) { h.has_sv2 = true; h.sv2 = typed_sort_value(cp.header.sort[1].kind, cp.sort_field_type[1], hits[i].v2); }
    r.partial_hits.push_back(std::move(h));
  }
  if (cp.header.num_aggs)
    r.intermediate_aggregation_result = hashed ? build_intermediate_aggs_entries(cp, img, entries, nentries) : build_intermediate_aggs(cp, img, cells, ncells);
  return r;
}

static void add_split_stats(pb::SplitResourceStats& a, const pb::SplitResourceStats& b) { for (int i = 0; i < 9; i++) a.v[i] += b.v[i]; }
static uint64_t phase_sum(const pb::SplitResourceStats& s) { return s.v[6] + s.v[8]; }  // warmup + cpu_search
static void add_leaf_stats(pb::LeafResourceStats& acc, const pb::LeafResourceStats& o) {
  acc.partial_result_cache_num_splits += o.partial_result_cache_num_splits;
  acc.partial_result_cache_num_docs += o.partial_result_cache_num_docs;
  acc.localexec_num_splits += o.localexec_num_splits;
  acc.localexec_num_docs += o.localexec_num_docs;
  acc.wall_time_microsecs += o.wall_time_microsecs;
  for (int i = 0; i < 5; i++) acc.lambda[i] += o.lambda[i];
  auto min_opt = [](std::optional<uint64_t> a, std::optional<uint64_t> b) { return !a ? b : (!b ? a : std::optional<uint64_t>(std::min(*a, *b))); };
  acc.min_wait_for_search_permit_microsecs = min_opt(acc.min_wait_for_search_permit_microsecs, o.min_wait_for_search_permit_microsecs);
  acc.min_wait_for_cpu_pool_microsecs = min_opt(acc.min_wait_for_cpu_pool_microsecs, o.min_wait_for_cpu_pool_microsecs);
  if (o.split_resources_sum) {
    if (!acc.split_resources_sum) acc.split_resources_sum = pb::SplitResourceStats();
    add_split_stats(*acc.split_resources_sum, *o.split_resources_sum);
  }
  if (o.split_resources_worst && (!acc.split_resources_worst || phase_sum(*o.split_resources_worst) >= phase_sum(*acc.split_resources_worst)))
    acc.split_resources_worst = o.split_resources_worst;
}

pb::LeafSearchResponse merge_responses(const pb::SearchRequest& req, std::vector<pb::LeafSearchResponse> parts) {
  int o1, o2;
  sort_orders(req, &o1, &o2);
  const size_t k = (size_t)(req.start_offset + req.max_hits);
  pb::LeafSearchResponse m;
  if (parts.size() == 1) {
    m = std::move(parts[0]);  // single-response shortcut (collector.rs:922-924)
  } else {
    std::vector<std::string> agg_parts;
    for (auto& p : parts) {
      if (p.resource_stats) { if (!m.resource_stats) m.resource_stats = pb::LeafResourceStats(); add_leaf_stats(*m.resource_stats, *p.resource_stats); }
      if (p.intermediate_aggregation_result) agg_parts.push_back(*p.intermediate_aggregation_result);
      m.num_attempted_splits += p.num_attempted_splits;
      m.num_successful_splits += p.num_successful_splits;
      m.num_hits += p.num_hits;
      for (auto& f : p.failed_splits) m.failed_splits.push_back(f);
    }
    if (req.aggregation_request && !req.aggregation_request->empty()) {
      std::vector<AggReq> reqs = parse_agg_request(*req.aggregation_request);
      m.intermediate_aggregation_result = merge_intermediate_aggs(reqs, agg_parts);
    }
    // top_k_partial_hits (collector.rs:980-992): TopK heap + sorted finalize == sort best-first, keep k.
    // Leaf responses arrive sorted best-first, so this is normally an n-way merge that stops after k
    // hits (ties go to the earlier part, like a stable sort of the concatenation); unsorted input falls
    // back to the sort.
    bool sorted = true;
    for (auto& p : parts)
      for (size_t i = 1; i < p.partial_hits.size() && sorted; i++)
        if (hit_cmp(o1, o2, p.partial_hits[i - 1], p.partial_hits[i]) < 0) sorted = false;
    if (sorted) {
      std::vector<size_t> pos(parts.size(), 0);
      while (m.partial_hits.size() < k) {
        int best = -1;
        for (size_t i = 0; i < parts.size(); i++) {
          if (pos[i] >= parts[i].partial_hits.size()) continue;
          if (best < 0 || hit_cmp(o1, o2, parts[i].partial_hits[pos[i]], parts[best].partial_hits[pos[best]]) > 0) best = (int)i;
        }
        if (best < 0) break;
        m.partial_hits.push_back(std::move(parts[best].partial_hits[pos[best]++]));
      }
    } else {
      for (auto& p : parts)
        for (auto& h : p.partial_hits) m.partial_hits.push_back(std::move(h));
      std::stable_sort(m.partial_hits.begin(), m.partial_hits.end(), [&](const pb::PartialHit& a, const pb::PartialHit& b) { return hit_cmp(o1, o2, a, b) > 0; });
      if (m.partial_hits.size() > k) m.partial_hits.resize(k);
    }
  }
  // merge_fruits: drop [..start_offset), truncate to max_hits (collector.rs:851-858)
  size_t drop = std::min<size_t>((size_t)req.start_offset, m.partial_hits.size());
  m.partial_hits.erase(m.partial_hits.begin(), m.partial_hits.begin() + drop);
  if (m.partial_hits.size() > req.max_hits) m.partial_hits.resize((size_t)req.max_hits);
  return m;
}

// ---- leaf search over the engine -------------------------------------------------------------------------
struct SplitJob {
  pb::SplitIdAndFooterOffsets meta;
  std::shared_ptr<SplitDev> dev;
  CompiledPlan plan;
  std::string error;
  int error_code = 0;
  bool metadata_count = false;  // answered from the split's num_docs alone (no plan, no device work)
  std::string cache_key;        // the split's partial-result cache key (empty: the cache is off)
  std::optional<std::string> cached;  // a cache hit: the split's encoded response (no plan, no device work)
};

struct LeafRun {
  std::vector<SplitJob> jobs;
  std::vector<size_t> which;      // jobs[which[k]] <-> outs[k]
  std::vector<uint32_t> id_rank;  // indexed like `jobs`: a searched split's rank by split id (breaks sort value ties)
  std::vector<SplitOutput> outs;
  BatchStats st;
  uint64_t wall_us = 0;
  bool merged_valid = false;       // the engine merged the per-split top-K lists on the device
  std::vector<MergedHit> merged;   // best-first; .split = index into `jobs` (gathered: global split rank)
  bool gathered = false;           // `merged` is the cross-rank result; rank_headers[r] = rank r's counters
  std::vector<RankHeader> rank_headers;
  bool use_cache = false;          // the partial-result cache was on for this call (no device merge: see §7.1)
};

static bool same_sort_types(const std::vector<SplitJob>& jobs, const std::vector<size_t>& which) {
  for (size_t k = 1; k < which.size(); k++) {
    const CompiledPlan &a = jobs[which[0]].plan, &b = jobs[which[k]].plan;
    for (int i = 0; i < 2; i++)
      if (a.header.sort[i].kind != b.header.sort[i].kind || (a.header.sort[i].kind == QW_SORT_COLUMN && a.sort_field_type[i] != b.sort_field_type[i] &&
                                                              a.header.sort[i].column != 0xFFFFFFFFu && b.header.sort[i].column != 0xFFFFFFFFu))
        return false;
  }
  return true;
}

// The sort kinds of the splits `which` (same_sort_types holds) and each key's sort-field type, taken from the first
// split that has the column (splits without it only produce None values)
struct SortTypes {
  uint32_t kind[2];
  int sft[2];
};
static SortTypes sort_types(const std::vector<SplitJob>& jobs, const std::vector<size_t>& which) {
  const CompiledPlan& p0 = jobs[which[0]].plan;
  SortTypes t = {{p0.header.sort[0].kind, p0.header.sort[1].kind}, {p0.sort_field_type[0], p0.sort_field_type[1]}};
  for (int i = 0; i < 2; i++)
    for (size_t w : which) {
      const CompiledPlan& p = jobs[w].plan;
      if (p.header.sort[i].kind == QW_SORT_COLUMN && p.header.sort[i].column != 0xFFFFFFFFu) { t.sft[i] = p.sort_field_type[i]; break; }
    }
  return t;
}
// A device-format hit of split `split_id` as a wire-form PartialHit (build_split_response's conversion)
static void append_hit(std::string& out, const std::string& split_id, const QwHit& h, const SortTypes& t) {
  pb::SortValue sv1, sv2;
  if (h.flags & 1) sv1 = typed_sort_value(t.kind[0], t.sft[0], h.v1);
  if (h.flags & 2) sv2 = typed_sort_value(t.kind[1], t.sft[1], h.v2);
  pb::append_partial_hit(out, 2, split_id, 0, h.doc_id, (h.flags & 1) != 0, sv1, (h.flags & 2) != 0, sv2);
}

// ---- pre-search pruning (SURVEY.md 8a row a16) ---------------------------------------------------------------
// CanSplitDoBetter::{from_request, optimize_split_order, optimize} (leaf.rs:1072-1242), is_simple_all_query
// (leaf.rs:1047-1069), disable_search_request_hits (leaf.rs:1438-1443), is_metadata_count_request_with_ast
// (root.rs:665-686). For a match-all request the split metadata alone says which splits can hold the top hits:
// the others are demoted to count-only requests, and a count-only match-all request without time bounds or
// aggregations is answered from `num_docs` without touching the split (leaf.rs:525-528).
// The reference also tightens the filter while the splits of a request run one after another
// (can_be_better / record_new_worst_hit, leaf.rs:1244-1285, 2012): the hits it removes are hits that cannot
// reach the top-K, so the response is the same; here all splits of a request run in one batch and that
// feedback has nothing to act on.
struct SplitFilter {
  enum Kind { Uninformative, SplitIdHigher, SplitTimestampHigher, SplitTimestampLower, FindTraceIdsAggregation } kind = Uninformative;
};
static bool is_trace_ids_on(const pb::SearchRequest& r, const std::string& timestamp_field) {
  if (r.max_hits != 0 || !r.aggregation_request || timestamp_field.empty()) return false;
  try {
    const std::vector<AggReq> a = parse_agg_request(*r.aggregation_request);
    return is_trace_ids_request(a) && a[0].ts_field == timestamp_field;
  } catch (const Error&) {
    return false;  // (a malformed request fails later, in compile_plan)
  }
}
static SplitFilter split_filter_from_request(const pb::SearchRequest& r, const std::string& timestamp_field) {
  SplitFilter f;
  // find_trace_ids over the index's timestamp field: the splits with the latest spans first (leaf.rs:1082-1090); they
  // are never skipped (leaf.rs:1420), which the aggregation request already guarantees below
  if (is_trace_ids_on(r, timestamp_field)) f.kind = SplitFilter::FindTraceIdsAggregation;
  else if (r.sort_fields.empty()) f.kind = SplitFilter::SplitIdHigher;
  else if (!timestamp_field.empty() && r.sort_fields[0].field_name == timestamp_field)
    f.kind = r.sort_fields[0].sort_order == 0 ? SplitFilter::SplitTimestampLower : SplitFilter::SplitTimestampHigher;
  return f;
}
static bool is_match_all_ast(const Json& ast) { return ast.type == Json::Obj && ast.str_or("type", "") == "match_all"; }
static bool is_simple_all_query(const pb::SearchRequest& r, const Json& ast) {
  if (r.aggregation_request || r.search_after || r.start_timestamp || r.end_timestamp) return false;
  return is_match_all_ast(ast);
}
static bool is_metadata_count_request(const pb::SearchRequest& r, const Json& ast) {
  return is_match_all_ast(ast) && r.max_hits == 0 && !r.start_timestamp && !r.end_timestamp && !r.aggregation_request && r.snippet_fields.empty();
}
static void disable_search_request_hits(pb::SearchRequest& r) {
  r.max_hits = 0;
  r.start_offset = 0;
  r.sort_fields.clear();
  r.search_after.reset();
}
struct SplitRequest {
  size_t input_pos;         // position of the split in the LeafRequestRef
  bool hits_disabled;       // demoted to a count-only request
  bool metadata_count;      // answered from num_docs
  bool skipped;             // simplify_search_request returned None: nothing to compute, the split is not searched
};
// the splits of one LeafRequestRef in the reference's processing order, with the per-split request rewrite
static std::vector<SplitRequest> optimize_split_requests(const pb::SearchRequest& r, const Json& ast, const std::string& timestamp_field,
                                                         const std::vector<pb::SplitIdAndFooterOffsets>& splits) {
  const SplitFilter f = split_filter_from_request(r, timestamp_field);
  auto ts_start = [&](size_t i) { return splits[i].timestamp_start.value_or(0); };  // prost getters: unset = 0
  auto ts_end = [&](size_t i) { return splits[i].timestamp_end.value_or(0); };
  std::vector<size_t> order(splits.size());
  for (size_t i = 0; i < order.size(); i++) order[i] = i;
  if (f.kind == SplitFilter::SplitIdHigher) std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return splits[a].split_id > splits[b].split_id; });
  else if (f.kind == SplitFilter::SplitTimestampHigher || f.kind == SplitFilter::FindTraceIdsAggregation) std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return ts_end(a) > ts_end(b); });
  else if (f.kind == SplitFilter::SplitTimestampLower) std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return ts_start(a) < ts_start(b); });
  std::vector<SplitRequest> out;
  for (size_t i : order) out.push_back({i, false, false, false});
  if (is_simple_all_query(r, ast)) {
    const uint64_t wanted = r.start_offset + r.max_hits;
    // splits guaranteed to deliver enough docs: the first prefix whose doc counts reach `wanted`
    size_t min_required = 1;
    uint64_t partial = 0;
    for (size_t k = 0; k < out.size(); k++) {
      partial += splits[out[k].input_pos].num_docs;
      if (partial < wanted) min_required++; else break;
    }
    if (f.kind == SplitFilter::SplitIdHigher) {
      for (size_t k = min_required; k < out.size(); k++) out[k].hits_disabled = true;
    } else if (f.kind == SplitFilter::SplitTimestampLower) {
      // only splits that start after every required split has ended cannot hold an earlier doc
      int64_t biggest_end = INT64_MIN;
      for (size_t k = 0; k < std::min(min_required, out.size()); k++) biggest_end = std::max(biggest_end, ts_end(out[k].input_pos));
      for (size_t k = min_required; k < out.size(); k++) if (ts_start(out[k].input_pos) > biggest_end) out[k].hits_disabled = true;
    } else if (f.kind == SplitFilter::SplitTimestampHigher) {
      int64_t smallest_start = INT64_MAX;
      for (size_t k = 0; k < std::min(min_required, out.size()); k++) smallest_start = std::min(smallest_start, ts_start(out[k].input_pos));
      for (size_t k = min_required; k < out.size(); k++) if (ts_end(out[k].input_pos) < smallest_start) out[k].hits_disabled = true;
    }
  }
  for (SplitRequest& q : out) {
    pb::SearchRequest rr = r;  // (only the fields the test reads)
    if (q.hits_disabled) disable_search_request_hits(rr);
    // simplify_search_request (leaf.rs:1399-1433): no hits wanted (any more), no aggregation, and the caller accepts an
    // underestimate of the hit count (CountHits::Underestimate = 1) => the split is pruned before warmup
    q.skipped = rr.max_hits == 0 && !rr.aggregation_request && r.count_hits == 1;
    q.metadata_count = !q.skipped && is_metadata_count_request(rr, ast);
  }
  return out;
}

// A failed split is reported retryable (leaf.rs:1989-2004: the root retries it on another node) unless the
// failure is a property of the request itself: a query shape or a top-K size this library does not execute
// fails the same way on every node, and retrying would only run it twice.
static inline bool retryable(int code) { return code != QWGPU_EUNSUPPORTED; }

// ---- partial-result cache (LeafSearchCache, leaf_cache.rs:27-185) ---------------------------------------------
// HalfOpenRange (leaf_cache.rs:120-185): [start, end), no end = unbounded above; every empty range normalises to 0..0
struct HalfOpenRange {
  int64_t start = 0;
  std::optional<int64_t> end;
  enum Bound { Unbounded, Included, Excluded };
  bool is_empty() const { return end && start >= *end; }  // !contains(start)
  HalfOpenRange normalize() const { return is_empty() ? HalfOpenRange{0, int64_t(0)} : *this; }
  static HalfOpenRange from_bounds(Bound sk, int64_t s, Bound ek, int64_t e) {
    HalfOpenRange r;
    if (sk == Included) r.start = s;
    else if (sk == Excluded) {
      if (s == INT64_MAX) return HalfOpenRange{0, int64_t(0)};  // excluding i64::MAX from below: empty
      r.start = s + 1;
    } else r.start = INT64_MIN;
    if (ek == Included) { if (e != INT64_MAX) r.end = e + 1; }  // including i64::MAX above: unbounded
    else if (ek == Excluded) r.end = e;
    return r.normalize();
  }
  HalfOpenRange intersect(const HalfOpenRange& o) const {
    HalfOpenRange r;
    r.start = std::max(start, o.start);
    r.end = end && o.end ? std::optional<int64_t>(std::min(*end, *o.end)) : (end ? end : o.end);
    return r.normalize();
  }
};

// CacheKey::from_split_meta_and_request (leaf_cache.rs:98-117): the split, the request without its time range and with
// count_hits = CountAll (at the scale of one split every hit is counted), and the merged time range: the request's
// [start_timestamp, end_timestamp) intersected with the split's [timestamp_start, timestamp_end]
// (SearchRequest::time_range / SplitIdAndFooterOffsets::time_range, quickwit-proto/src/search/mod.rs:33-51). So a
// window that covers the whole split keys like any other window that does. Requests compare by their encoded bytes.
// The reference keys on the split id alone; here every request carries its own doc mapper, and the doc mapper decides
// how the split is read (fields, tokenizers, the timestamp field), so the doc mapper string is part of the key: a
// split searched through a changed mapper must not hit the entry of the old one. It costs nothing while a split's
// mapper stays the same.
static std::string leaf_cache_key(const pb::SplitIdAndFooterOffsets& split, pb::SearchRequest req, const std::string& doc_mapper,
                                  HalfOpenRange* range_out = nullptr) {
  using R = HalfOpenRange;
  const R split_range = R::from_bounds(split.timestamp_start ? R::Included : R::Unbounded, split.timestamp_start.value_or(0),
                                       split.timestamp_end ? R::Included : R::Unbounded, split.timestamp_end.value_or(0));
  const R req_range = R::from_bounds(req.start_timestamp ? R::Included : R::Unbounded, req.start_timestamp.value_or(0),
                                     req.end_timestamp ? R::Excluded : R::Unbounded, req.end_timestamp.value_or(0));
  const R merged = req_range.intersect(split_range);
  if (range_out) *range_out = merged;
  req.start_timestamp.reset();
  req.end_timestamp.reset();
  req.count_hits = 0;  // CountHits::CountAll
  std::string key;
  auto field = [&](const std::string& b) {
    const uint64_t n = b.size();
    key.append((const char*)&n, 8);
    key += b;
  };
  field(split.split_id);
  field(doc_mapper);
  field(pb::encode_search_request(req));
  const int64_t r[3] = {merged.start, merged.end ? 1 : 0, merged.end.value_or(0)};
  key.append((const char*)r, sizeof r);
  return key;
}

bool LeafCache::get(const std::string& key, std::string* value) {
  std::lock_guard<std::mutex> g(mu);
  auto it = index.find(key);
  if (it == index.end()) { misses++; return false; }
  hits++;
  lru.splice(lru.begin(), lru, it->second);
  *value = it->second->value;
  return true;
}

void LeafCache::put(const std::string& split_id, const std::string& key, std::string value) {
  std::lock_guard<std::mutex> g(mu);
  if (value.size() > budget) return;  // (also when the cache is off) MemorySizedCache drops what exceeds its capacity
  auto it = index.find(key);
  if (it != index.end()) {  // (a concurrent call filled the same key first: the newer value replaces it)
    used -= it->second->value.size();
    lru.erase(it->second);
    index.erase(it);
  }
  while (used + value.size() > budget) {
    used -= lru.back().value.size();
    index.erase(lru.back().key);
    lru.pop_back();
    evictions++;
  }
  used += value.size();
  lru.push_front(Entry{key, split_id, std::move(value)});
  index[key] = lru.begin();
  fills++;
}

void LeafCache::set_budget(uint64_t bytes) {
  std::lock_guard<std::mutex> g(mu);
  budget = bytes;
  while (used > budget) {
    used -= lru.back().value.size();
    index.erase(lru.back().key);
    lru.pop_back();
    evictions++;
  }
}

void LeafCache::drop_split(const std::string& split_id) {
  std::lock_guard<std::mutex> g(mu);
  for (auto it = lru.begin(); it != lru.end();) {
    if (it->split_id != split_id) { ++it; continue; }
    used -= it->value.size();
    index.erase(it->key);
    it = lru.erase(it);
  }
}

// LeafSearchCache::put (leaf_cache.rs:66-80): the split's response with its resource stats replaced by the cache-hit
// counters, so that a hit reports itself
static std::string cache_value(const SplitJob& j, pb::LeafSearchResponse r) {
  pb::LeafResourceStats s;
  s.partial_result_cache_num_splits = 1;
  s.partial_result_cache_num_docs = j.meta.num_docs;
  r.resource_stats = s;
  return pb::encode_leaf_search_response(r);
}

// Stores the (job index, cache_value) pairs of one call. Only successful searches come here (leaf.rs:695-705 stores
// the response of leaf_search_single_split when a search ran; a failed, pruned or metadata-count split stores
// nothing). A value is kept only while its split id still names the image it was computed on: under Engine::mu,
// against the registration that drops the split's entries (Engine::register_split / unregister_split).
static void store_responses(Engine& eng, const LeafRun& run, std::vector<std::pair<size_t, std::string>> values) {
  if (values.empty()) return;
  std::lock_guard<std::mutex> g(eng.mu);
  for (auto& v : values) {
    const SplitJob& j = run.jobs[v.first];
    auto it = eng.splits.find(j.meta.split_id);
    if (it != eng.splits.end() && it->second == j.dev) eng.leaf.put(j.meta.split_id, j.cache_key, std::move(v.second));
  }
}

// add_top_cache_node (rewrite_request, leaf.rs:724-737): a request with search_after is a page of a paged search, and
// the pages after it evaluate the same query again. With the context's predicate cache enabled, the query AST is
// wrapped in a `cache` node, so that each split's doc set is computed once and read by every later page. A request
// ranked by _score compiles the node as its inner query (compile_plan); with the cache disabled nothing is wrapped.
// Like the reference, which wraps each split's request after the split-level decisions (optimize_split_requests reads
// the AST unwrapped), the wrapped AST `out` only goes to the compiler. False: not wrapped.
static bool add_top_cache_node(Engine& eng, const Json& ast, Json& out) {
  {
    std::lock_guard<std::mutex> g(eng.pred.mu);
    if (!eng.pred.budget) return false;
  }
  Json type;
  type.type = Json::Str;
  type.s = "cache";
  out = Json();
  out.type = Json::Obj;
  out.obj.emplace_back("type", std::move(type));
  out.obj.emplace_back("inner", ast);
  return true;
}

static void run_leaf_raw(Engine& eng, const pb::LeafSearchRequest& lr, LeafRun& run, bool want_merged = false, const Comm* comm = nullptr) {
  using clock = std::chrono::steady_clock;
  const pb::SearchRequest& sreq = lr.search_request;
  const auto t_compile = clock::now();
  Json ast = parse_json(sreq.query_ast, QWGPU_EINVALID_QUERY);  // once per request
  Json cached_ast;
  const Json* compile_ast = sreq.search_after && add_top_cache_node(eng, ast, cached_ast) ? &cached_ast : &ast;
  // the partial-result cache (process_partial_result_cache, leaf.rs:1872-1896): a split is looked up after its request
  // rewrite and before warmup, so a hit needs neither the split's residency nor a plan. The NCCL road builds its
  // exchanged record on the device and bypasses the cache. With the cache on, each searched split's own response is
  // stored, so the per-split lists come back instead of the device merge's list (DESIGN.md §7.1).
  run.use_cache = !comm && eng.leaf.on();
  if (run.use_cache) want_merged = false;
  for (auto& ref : lr.leaf_requests) {
    if (ref.doc_mapper_ord >= lr.doc_mappers.size()) fail(QWGPU_EINVALID_ARG, "Internal error: doc_mapper_ord out of bounds");
    DocMapperInfo dm = parse_doc_mapper(lr.doc_mappers[ref.doc_mapper_ord]);
    // per-split request rewrite (a16); the jobs keep the request's split order (the processing order of a
    // batch is not observable). Across ranks every split goes to the device: the counters of the exchanged
    // record are built there.
    std::vector<SplitRequest> opt = optimize_split_requests(sreq, ast, dm.timestamp_field, ref.split_offsets);
    std::vector<const SplitRequest*> by_pos(ref.split_offsets.size(), nullptr);
    for (const SplitRequest& q : opt) by_pos[q.input_pos] = &q;
    pb::SearchRequest count_req;
    bool have_count_req = false;
    for (size_t si = 0; si < ref.split_offsets.size(); si++) {
      const pb::SplitIdAndFooterOffsets& so = ref.split_offsets[si];
      const SplitRequest& q = *by_pos[si];
      if (q.skipped && !comm) continue;  // (PrunedBeforeWarmup: contributes nothing, not even to the split counters)
      SplitJob j;
      j.meta = so;
      if (q.metadata_count && !comm) {
        j.metadata_count = true;
        run.jobs.push_back(std::move(j));
        continue;
      }
      const pb::SearchRequest* req = &sreq;
      if (q.hits_disabled) {
        if (!have_count_req) { count_req = sreq; disable_search_request_hits(count_req); have_count_req = true; }
        req = &count_req;
      }
      if (run.use_cache) {
        j.cache_key = leaf_cache_key(so, *req, lr.doc_mappers[ref.doc_mapper_ord]);
        std::string v;
        if (eng.leaf.get(j.cache_key, &v)) {
          j.cached = std::move(v);
          run.jobs.push_back(std::move(j));
          continue;
        }
      }
      j.dev = eng.find(so.split_id);
      try {
        if (!j.dev) fail(QWGPU_ENOTFOUND, "split `%s` is not resident on this GPU", so.split_id.c_str());
        j.plan = compile_plan(j.dev->view, so.split_id, *req, dm, &so, compile_ast);
      } catch (const Error& e) {
        // malformed queries / aggregations fail the whole request like the reference (service.rs:182-184); so does
        // a query or aggregation shape this library does not compile: every split would fail the same way
        if (e.code == QWGPU_EINVALID_QUERY || e.code == QWGPU_EINVALID_AGG || e.code == QWGPU_EINVALID_ARG || e.code == QWGPU_EUNSUPPORTED) throw;
        j.error = e.what();
        j.error_code = e.code;
      }
      run.jobs.push_back(std::move(j));
    }
  }
  std::vector<std::shared_ptr<SplitDev>> devs;
  std::vector<const uint8_t*> plans;
  std::vector<size_t> lens;
  for (size_t i = 0; i < run.jobs.size(); i++)
    if (!run.jobs[i].error_code && !run.jobs[i].metadata_count && !run.jobs[i].cached) {
      devs.push_back(run.jobs[i].dev);
      plans.push_back((const uint8_t*)run.jobs[i].plan.bytes.data());
      lens.push_back(run.jobs[i].plan.bytes.size());
      run.which.push_back(i);
    }
  std::vector<size_t> by_id(run.which);
  std::sort(by_id.begin(), by_id.end(), [&](size_t a, size_t b) { return run.jobs[a].meta.split_id < run.jobs[b].meta.split_id; });
  run.id_rank.assign(run.jobs.size(), 0);
  for (size_t r = 0; r < by_id.size(); r++) run.id_rank[by_id[r]] = (uint32_t)r;
  auto t0 = clock::now();
  if (getenv("QWGPU_TRACE"))
    fprintf(stderr, "[qwgpu] compile: %ld us for %zu splits\n", (long)std::chrono::duration_cast<std::chrono::microseconds>(t0 - t_compile).count(), run.jobs.size());
  MergeSpec ms;
  GatherSpec gs;
  const bool gathering = comm && comm->world > 1 && sreq.max_hits + sreq.start_offset > 0;
  if (gathering && !same_sort_types(run.jobs, run.which)) fail(QWGPU_EUNSUPPORTED, "the splits of this rank disagree on the sort field types: cross-rank merge on the device is not possible");
  if ((gathering || (want_merged && devs.size() > 1)) && sreq.max_hits + sreq.start_offset > 0 && same_sort_types(run.jobs, run.which)) {
    int o1, o2;
    sort_orders(sreq, &o1, &o2);
    ms.k = (uint32_t)(sreq.max_hits + sreq.start_offset);
    ms.order1 = (uint32_t)o1; ms.order2 = (uint32_t)o2;
    const size_t n = run.which.size();
    ms.rank.resize(n);
    for (size_t i = 0; i < n; i++) ms.rank[i] = run.id_rank[run.which[i]];
    if (gathering) {
      // tie-breaks across ranks use the split id order of the WHOLE query: ranks from the context's table
      for (size_t i = 0; i < n; i++) {
        const int g = comm_split_rank(comm, run.jobs[run.which[i]].meta.split_id);
        if (g < 0) fail(QWGPU_EINVALID_ARG, "split `%s` is not in the communicator's split table (qwgpu_comm_set_split_table)", run.jobs[run.which[i]].meta.split_id.c_str());
        ms.rank[i] = (uint32_t)g;
      }
      gs.world = comm->world; gs.rank = comm->rank; gs.allgather = comm_allgather; gs.comm = comm->comm;
      gs.attempted = run.jobs.size(); gs.successful = devs.size(); gs.n_failed = run.jobs.size() - devs.size();
    }
  }
  if (!devs.empty() || gathering)
    eng.search(devs, plans, lens, run.outs, run.st, ms.k ? &ms : nullptr, ms.k ? &run.merged : nullptr, gathering ? &gs : nullptr, gathering ? &run.rank_headers : nullptr);
  if (gathering) run.gathered = true;
  else if (ms.k) {
    run.merged_valid = true;
    for (auto& m : run.merged) m.split = (uint32_t)run.which[m.split];
  }
  run.wall_us = (uint64_t)std::chrono::duration_cast<std::chrono::microseconds>(clock::now() - t0).count();
}

// SplitResourceStats / LeafResourceStats filled like leaf.rs:641-684; cpu_search_microsecs carries the
// split's share of the batch's device time
static pb::LeafResourceStats split_stats(const LeafRun& run, size_t k) {
  const SplitJob& j = run.jobs[run.which[k]];
  const size_t n = std::max<size_t>(run.which.size(), 1);
  pb::SplitResourceStats ss;
  ss.v[0] = j.dev->view.hdr->num_docs;
  ss.v[1] = j.dev->data_len;
  ss.v[4] = run.outs[k].num_hits;
  ss.v[8] = (uint64_t)(run.st.gpu_time_us / n);
  pb::LeafResourceStats ls;
  ls.localexec_num_splits = 1;
  ls.localexec_num_docs = ss.v[0];
  ls.split_resources_sum = ss;
  ls.split_resources_worst = ss;
  ls.min_wait_for_search_permit_microsecs = 0;
  ls.min_wait_for_cpu_pool_microsecs = 0;
  ls.wall_time_microsecs = run.wall_us / n;
  return ls;
}

static std::vector<pb::LambdaSingleSplitResult> run_leaf(Engine& eng, const pb::LeafSearchRequest& lr) {
  LeafRun run;
  run_leaf_raw(eng, lr, run);
  std::vector<pb::LambdaSingleSplitResult> results(run.jobs.size());
  for (size_t i = 0; i < run.jobs.size(); i++) {
    results[i].split_id = run.jobs[i].meta.split_id;
    if (run.jobs[i].error_code) { results[i].is_error = true; results[i].error = run.jobs[i].error; }
    if (run.jobs[i].metadata_count) {  // get_leaf_resp_from_count (leaf.rs:474-484)
      pb::LeafSearchResponse r;
      r.num_hits = run.jobs[i].meta.num_docs;
      r.num_attempted_splits = r.num_successful_splits = 1;
      results[i].response = std::move(r);
    }
  }
  for (size_t i = 0; i < run.jobs.size(); i++)
    if (run.jobs[i].cached) results[i].response = pb::decode_leaf_search_response((const uint8_t*)run.jobs[i].cached->data(), run.jobs[i].cached->size());
  std::vector<std::pair<size_t, std::string>> fills;
  for (size_t k = 0; k < run.which.size(); k++) {
    size_t i = run.which[k];
    SplitOutput& o = run.outs[k];
    if (o.status) { results[i].is_error = true; results[i].error = o.error; continue; }
    pb::LeafSearchResponse r = build_split_response(run.jobs[i].plan, run.jobs[i].dev->view, run.jobs[i].meta.split_id, o.num_hits,
                                                    o.hits.data(), o.hits.size(), o.cells.data(), o.cells.size(),
                                                    o.entries.data(), o.entries.size(), o.hashed);
    if (run.use_cache) fills.emplace_back(i, cache_value(run.jobs[i], r));
    r.resource_stats = split_stats(run, k);
    results[i].response = std::move(r);
  }
  store_responses(eng, run, std::move(fills));
  return results;
}

// Leaf-level merge (IncrementalCollector, collector.rs:1195-1313) done on the device-format hits: the
// per-split lists are already sorted best-first, so a k-way heap merge in the u64 fast-field space
// (order-preserving per sort-field type) yields the leaf's top (max_hits + start_offset) without
// materialising every split's PartialHits. Falls back to the generic path when the sort-field types
// differ across splits.
static pb::LeafSearchResponse leaf_merge_fast(const pb::SearchRequest& sreq, LeafRun& run) {
  pb::LeafSearchResponse m;
  const size_t n = run.which.size();
  int o1, o2;
  sort_orders(sreq, &o1, &o2);
  const size_t k = (size_t)(sreq.max_hits + sreq.start_offset);
  const SortTypes types = sort_types(run.jobs, run.which);
  // Heads of the per-split lists as plain integer tuples, greater = better: (has1, v1', has2, v2', tie')
  // with v' = v for a descending key and ~v for an ascending one (None — has = 0 — is last in both
  // directions, compare_opt in quickwit-proto/src/lib.rs:122-140), tie' = (split rank, doc id) in the
  // direction of the first key (collector.rs:1120-1153). Built only for the current head of each list.
  struct Head {
    uint64_t v1, v2, tie;
    uint32_t s;
    uint8_t has1, has2;
    bool operator<(const Head& o) const { return std::tie(has1, v1, has2, v2, tie) < std::tie(o.has1, o.v1, o.has2, o.v2, o.tie); }
  };
  auto head_of = [&](size_t sidx, const QwHit& h) {
    Head k;
    k.s = (uint32_t)sidx;
    k.has1 = h.flags & 1;
    k.has2 = (h.flags >> 1) & 1;
    k.v1 = k.has1 ? (o1 == QW_ORDER_DESC ? h.v1 : ~h.v1) : 0;
    k.v2 = k.has2 ? (o2 == QW_ORDER_DESC ? h.v2 : ~h.v2) : 0;
    const uint64_t t = ((uint64_t)run.id_rank[run.which[sidx]] << 32) | h.doc_id;
    k.tie = o1 == QW_ORDER_DESC ? t : ~t;
    return k;
  };
  std::vector<size_t> pos(n, 0);
  std::vector<Head> heap;
  std::vector<SplitAggCells> agg_parts;
  pb::LeafResourceStats stats_acc;
  bool any_stats = false;
  for (size_t s = 0; s < n; s++) {
    SplitOutput& o = run.outs[s];
    m.num_hits += o.num_hits;
    m.num_attempted_splits += 1;
    m.num_successful_splits += 1;
    if (!o.hits.empty()) heap.push_back(head_of(s, o.hits[0]));
    const SplitJob& j = run.jobs[run.which[s]];
    if (j.plan.header.num_aggs)
      agg_parts.push_back({&j.plan, &j.dev->view, o.cells.data(), o.cells.size(), o.hashed, o.entries.data(), o.entries.size()});
    add_leaf_stats(stats_acc, split_stats(run, s));
    any_stats = true;
  }
  std::make_heap(heap.begin(), heap.end());
  // the merged hits go straight to wire form (no PartialHit temporaries: a split id is a 26-char ULID)
  size_t taken = 0;
  m.encoded_partial_hits.reserve(std::min<size_t>(k, 4096) * 72);
  if (run.merged_valid) {
    // the engine already merged on the device (k_merge): same total order, hits arrive best-first
    for (const MergedHit& mh : run.merged) {
      if (taken >= k) break;
      append_hit(m.encoded_partial_hits, run.jobs[mh.split].meta.split_id, mh.hit, types);
      taken++;
    }
    heap.clear();
  }
  while (!heap.empty() && taken < k) {
    std::pop_heap(heap.begin(), heap.end());
    size_t s = heap.back().s;
    append_hit(m.encoded_partial_hits, run.jobs[run.which[s]].meta.split_id, run.outs[s].hits[pos[s]], types);
    taken++;
    if (++pos[s] < run.outs[s].hits.size()) { heap.back() = head_of(s, run.outs[s].hits[pos[s]]); std::push_heap(heap.begin(), heap.end()); }
    else heap.pop_back();
  }
  if (sreq.aggregation_request && !sreq.aggregation_request->empty())
    m.intermediate_aggregation_result = build_and_merge_intermediate_aggs(run.jobs[run.which[0]].plan.agg_request, agg_parts);
  if (any_stats) m.resource_stats = stats_acc;
  return m;
}

// The leaf merge with the partial-result cache on: each searched split's own response is built and stored, and merged
// with the cached responses through merge_responses (the IncrementalCollector takes cached and searched responses
// alike, leaf.rs:1872-1896). The parts keep the request's split order, the order in which leaf_merge_fast folds the
// same splits' aggregations, so an aggregation merges the same f64 values in the same order with and without the
// cache. `run` holds the successful searches only.
static pb::LeafSearchResponse leaf_merge_cached(Engine& eng, const pb::SearchRequest& mreq, LeafRun& run) {
  std::vector<int> slot(run.jobs.size(), -1);
  for (size_t k = 0; k < run.which.size(); k++) slot[run.which[k]] = (int)k;
  std::vector<pb::LeafSearchResponse> parts;
  std::vector<std::pair<size_t, std::string>> fills;
  for (size_t i = 0; i < run.jobs.size(); i++) {
    const SplitJob& j = run.jobs[i];
    if (j.cached) {
      parts.push_back(pb::decode_leaf_search_response((const uint8_t*)j.cached->data(), j.cached->size()));
      continue;
    }
    if (slot[i] < 0) continue;  // failed, or answered from the split's metadata
    const size_t k = (size_t)slot[i];
    const SplitOutput& o = run.outs[k];
    pb::LeafSearchResponse r = build_split_response(j.plan, j.dev->view, j.meta.split_id, o.num_hits, o.hits.data(), o.hits.size(),
                                                    o.cells.data(), o.cells.size(), o.entries.data(), o.entries.size(), o.hashed);
    fills.emplace_back(i, cache_value(j, r));
    r.resource_stats = split_stats(run, k);
    parts.push_back(std::move(r));
  }
  store_responses(eng, run, std::move(fills));
  pb::LeafSearchResponse m;
  if (!parts.empty()) m = merge_responses(mreq, std::move(parts));
  else if (mreq.aggregation_request && !mreq.aggregation_request->empty())
    m.intermediate_aggregation_result = merge_intermediate_aggs(parse_agg_request(*mreq.aggregation_request), {});
  return m;
}

}  // namespace qw

// ---- C ABI --------------------------------------------------------------------------------------------------
#define QW_API_BEGIN try {
#define QW_API_END                                   \
  }                                                  \
  catch (const qw::Error& e) {                       \
    qw::set_last_error(e.what());                    \
    return e.code;                                   \
  }                                                  \
  catch (const std::exception& e) {                  \
    qw::set_last_error(e.what());                    \
    return QWGPU_EINTERNAL;                          \
  }

static void give(const std::string& s, uint8_t** out, size_t* len) {
  *out = (uint8_t*)malloc(s.size() ? s.size() : 1);
  if (!*out) qw::fail(QWGPU_EINTERNAL, "out of memory");
  memcpy(*out, s.data(), s.size());
  *len = s.size();
}
static qw::Engine& engine_of(qwgpu_ctx* ctx) {
  if (!ctx) qw::fail(QWGPU_EINVALID_ARG, "null context");
  if (!ctx->engine) qw::fail(QWGPU_ENODEVICE, "host-only context: no CUDA device bound (there is no CPU search path)");
  return *ctx->engine;
}

// the split image opened into `v`, and the search request's plan on it
static qw::CompiledPlan host_compile(qw::ImageView& v, const uint8_t* img, uint64_t img_len, const char* split_id,
                                     const uint8_t* search_request_pb, size_t search_request_len, const char* doc_mapper_json) {
  v.open(img, img_len);
  qw::pb::SearchRequest req = qw::pb::decode_search_request(qw::pb::Reader(search_request_pb, search_request_len));
  qw::DocMapperInfo dm = qw::parse_doc_mapper(doc_mapper_json ? doc_mapper_json : "");
  return qw::compile_plan(v, split_id ? split_id : "", req, dm, nullptr);
}

namespace {
// fixed-size per-rank partial for the single all-gather (SURVEY.md §8e):
//   [u64 magic][u64 num_hits][u64 attempted][u64 successful][u32 n_hits][u32 agg_len][u32 n_failed][u32 pad]
//   n_hits x [u8 kind1, u8 kind2, u16 split_len, u32 doc_id, u64 v1, u64 v2, char split_id[40]]
//   tail (kTailCap reserved): LeafSearchResponse{failed_splits, resource_stats}
//   agg bytes (<= kAggCap) — last, so that the used part of a partial is a prefix of it (partial_used_bytes)
const uint64_t kPartMagic = 0x5452415057515157ull;
const size_t kHitBytes = 64, kAggCap = 1 << 20, kTailCap = 4096;
static_assert(kAggCap >= (size_t)QW_MAX_TOPK * 26 + 5, "a partial holds the largest find_trace_ids result (N spans of <= 26 bytes + length)");
uint64_t partial_bytes_for(const qw::pb::SearchRequest& r) {
  size_t k = (size_t)(r.max_hits + r.start_offset);
  bool aggs = r.aggregation_request && !r.aggregation_request->empty();
  return 48 + k * kHitBytes + (aggs ? kAggCap : 0) + kTailCap;
}
// bytes of a filled partial that carry information (a prefix): header, hit slots, tail, the aggregation bytes in use
uint64_t partial_used_bytes(const qw::pb::SearchRequest& r, const uint8_t* partial) {
  uint32_t meta[4];
  memcpy(meta, partial + 32, 16);
  return 48 + (size_t)(r.max_hits + r.start_offset) * kHitBytes + kTailCap + std::min<size_t>(meta[1], kAggCap);
}
}  // namespace

extern "C" {

int qwgpu_leaf_search(qwgpu_ctx* ctx, const uint8_t* req, size_t req_len, uint8_t** resp, size_t* resp_len) {
  QW_API_BEGIN
  qw::Engine& eng = engine_of(ctx);
  // QWGPU_TRACE=1: per-phase host timings of this call on stderr (diagnostics only)
  static const bool trace = getenv("QWGPU_TRACE") != nullptr;
  using tclock = std::chrono::steady_clock;
  auto t_start = tclock::now();
  qw::pb::LeafSearchRequest lr = qw::pb::decode_leaf_search_request(req, req_len);
  auto t_dec = tclock::now();
  qw::LeafRun run;
  qw::run_leaf_raw(eng, lr, run, /*want_merged=*/true);
  auto t_run = tclock::now();
  // the leaf keeps [0, start_offset + max_hits) (root.rs:1775-1777): nothing is drained here
  qw::pb::SearchRequest mreq = lr.search_request;
  mreq.max_hits += mreq.start_offset;
  mreq.start_offset = 0;
  std::vector<qw::pb::SplitSearchError> failed;
  for (auto& j : run.jobs) if (j.error_code) failed.push_back({j.error, j.meta.split_id, qw::retryable(j.error_code)});
  // drop splits whose search failed on the device from the merge set
  {
    std::vector<size_t> w2;
    std::vector<qw::SplitOutput> o2;
    for (size_t k = 0; k < run.which.size(); k++) {
      if (run.outs[k].status) failed.push_back({run.outs[k].error, run.jobs[run.which[k]].meta.split_id, qw::retryable(run.outs[k].status)});
      else { w2.push_back(run.which[k]); o2.push_back(std::move(run.outs[k])); }
    }
    run.which.swap(w2);
    run.outs.swap(o2);
  }
  const bool same_types = run.merged_valid || qw::same_sort_types(run.jobs, run.which);
  qw::pb::LeafSearchResponse merged;
  if (run.use_cache) {
    merged = qw::leaf_merge_cached(eng, mreq, run);
  } else if (run.which.empty()) {
    if (mreq.aggregation_request && !mreq.aggregation_request->empty())
      merged.intermediate_aggregation_result = qw::merge_intermediate_aggs(qw::parse_agg_request(*mreq.aggregation_request), {});
  } else if (same_types) {
    merged = qw::leaf_merge_fast(mreq, run);
  } else {
    std::vector<qw::pb::LeafSearchResponse> parts;
    for (size_t k = 0; k < run.which.size(); k++) {
      const qw::SplitJob& j = run.jobs[run.which[k]];
      qw::SplitOutput& o = run.outs[k];
      qw::pb::LeafSearchResponse r = qw::build_split_response(j.plan, j.dev->view, j.meta.split_id, o.num_hits, o.hits.data(), o.hits.size(), o.cells.data(), o.cells.size(),
                                                              o.entries.data(), o.entries.size(), o.hashed);
      r.resource_stats = qw::split_stats(run, k);
      parts.push_back(std::move(r));
    }
    merged = parts.size() == 1 ? std::move(parts[0]) : qw::merge_responses(mreq, std::move(parts));
  }
  for (auto& f : failed) { merged.failed_splits.push_back(f); merged.num_attempted_splits += 1; }
  for (auto& j : run.jobs)
    if (j.metadata_count) {  // get_leaf_resp_from_count (leaf.rs:474-484) merged in: counters only
      merged.num_hits += j.meta.num_docs;
      merged.num_attempted_splits += 1;
      merged.num_successful_splits += 1;
    }
  auto t_merge = tclock::now();
  give(qw::pb::encode_leaf_search_response(merged), resp, resp_len);
  if (trace) {
    auto us = [](tclock::time_point a, tclock::time_point b) { return (long)std::chrono::duration_cast<std::chrono::microseconds>(b - a).count(); };
    size_t cached = 0;
    for (auto& j : run.jobs) cached += j.cached ? 1 : 0;
    fprintf(stderr, "[qwgpu] leaf_search: decode %ld us, compile+search %ld us (engine wall %lu us, device %.0f us, %u launches, %zu splits from the cache), merge %ld us, encode %ld us\n",
            us(t_start, t_dec), us(t_dec, t_run), (unsigned long)run.wall_us, run.st.gpu_time_us, run.st.launches, cached, us(t_run, t_merge), us(t_merge, tclock::now()));
  }
  return 0;
  QW_API_END
}

// Host only: the per-split request rewrite of a LeafSearchRequest as JSON, in the reference's processing order:
// [{"split_id", "max_hits", "hits_disabled", "metadata_count", "skipped"} ...] per LeafRequestRef (concatenated).
int qwgpu_optimize_leaf_request(const uint8_t* req, size_t req_len, uint8_t** out, size_t* out_len) {
  QW_API_BEGIN
  if (!req || !out || !out_len) qw::fail(QWGPU_EINVALID_ARG, "null argument");
  qw::pb::LeafSearchRequest lr = qw::pb::decode_leaf_search_request(req, req_len);
  qw::Json ast = qw::parse_json(lr.search_request.query_ast, QWGPU_EINVALID_QUERY);
  std::string js = "[";
  for (auto& ref : lr.leaf_requests) {
    if (ref.doc_mapper_ord >= lr.doc_mappers.size()) qw::fail(QWGPU_EINVALID_ARG, "Internal error: doc_mapper_ord out of bounds");
    qw::DocMapperInfo dm = qw::parse_doc_mapper(lr.doc_mappers[ref.doc_mapper_ord]);
    for (const qw::SplitRequest& q : qw::optimize_split_requests(lr.search_request, ast, dm.timestamp_field, ref.split_offsets)) {
      if (js.size() > 1) js += ",";
      std::string id;
      for (char c : ref.split_offsets[q.input_pos].split_id) { if (c == '"' || c == '\\') id += '\\'; id += c; }
      js += "{\"split_id\":\"" + id + "\",\"max_hits\":" + std::to_string(q.hits_disabled ? 0 : lr.search_request.max_hits) +
            ",\"hits_disabled\":" + (q.hits_disabled ? "true" : "false") + ",\"metadata_count\":" + (q.metadata_count ? "true" : "false") +
            ",\"skipped\":" + (q.skipped ? "true" : "false") + "}";
    }
  }
  js += "]";
  give(js, out, out_len);
  return 0;
  QW_API_END
}

// Host only: the partial-result cache key of every split of a LeafSearchRequest as JSON, in the reference's processing
// order: [{"split_id", "looked_up", "key" (hex), "range": [start, end or null]} ...] per LeafRequestRef (concatenated).
// looked_up: false for a split that is pruned or answered from its metadata, which the cache never sees.
int qwgpu_leaf_cache_keys(const uint8_t* req, size_t req_len, uint8_t** out, size_t* out_len) {
  QW_API_BEGIN
  if (!req || !out || !out_len) qw::fail(QWGPU_EINVALID_ARG, "null argument");
  qw::pb::LeafSearchRequest lr = qw::pb::decode_leaf_search_request(req, req_len);
  qw::Json ast = qw::parse_json(lr.search_request.query_ast, QWGPU_EINVALID_QUERY);
  std::string js = "[";
  for (auto& ref : lr.leaf_requests) {
    if (ref.doc_mapper_ord >= lr.doc_mappers.size()) qw::fail(QWGPU_EINVALID_ARG, "Internal error: doc_mapper_ord out of bounds");
    qw::DocMapperInfo dm = qw::parse_doc_mapper(lr.doc_mappers[ref.doc_mapper_ord]);
    for (const qw::SplitRequest& q : qw::optimize_split_requests(lr.search_request, ast, dm.timestamp_field, ref.split_offsets)) {
      const qw::pb::SplitIdAndFooterOffsets& so = ref.split_offsets[q.input_pos];
      qw::pb::SearchRequest rr = lr.search_request;
      if (q.hits_disabled) qw::disable_search_request_hits(rr);
      qw::HalfOpenRange range;
      const std::string key = qw::leaf_cache_key(so, rr, lr.doc_mappers[ref.doc_mapper_ord], &range);
      std::string hex, id;
      for (unsigned char c : key) { hex += "0123456789abcdef"[c >> 4]; hex += "0123456789abcdef"[c & 15]; }
      for (char c : so.split_id) { if (c == '"' || c == '\\') id += '\\'; id += c; }
      if (js.size() > 1) js += ",";
      js += "{\"split_id\":\"" + id + "\",\"looked_up\":" + (q.skipped || q.metadata_count ? "false" : "true") + ",\"key\":\"" + hex +
            "\",\"range\":[" + std::to_string(range.start) + "," + (range.end ? std::to_string(*range.end) : "null") + "]}";
    }
  }
  js += "]";
  give(js, out, out_len);
  return 0;
  QW_API_END
}

// ---- collectives (comm.cpp) ----------------------------------------------------------------------------------
int qwgpu_comm_unique_id(uint8_t* out128) {
  QW_API_BEGIN
  if (!out128) qw::fail(QWGPU_EINVALID_ARG, "null out pointer");
  qw::comm_unique_id(out128);
  return 0;
  QW_API_END
}
int qwgpu_comm_init_lane(qwgpu_ctx* ctx, uint32_t lane, const uint8_t* id128, int rank, int world) {
  QW_API_BEGIN
  qw::Engine& eng = engine_of(ctx);
  if (!id128) qw::fail(QWGPU_EINVALID_ARG, "null unique id");
  if (lane >= 16) qw::fail(QWGPU_EINVALID_ARG, "lane %u (at most 16 lanes)", lane);
  if (ctx->lanes[lane]) { qw::comm_destroy(ctx->lanes[lane]); ctx->lanes[lane] = nullptr; }
  ctx->lanes[lane] = qw::comm_create(eng.device, id128, rank, world);
  if (lane && ctx->lanes[0]) ctx->lanes[lane]->split_ids = ctx->lanes[0]->split_ids;
  ctx->comm = ctx->lanes[0];
  return 0;
  QW_API_END
}
int qwgpu_comm_init(qwgpu_ctx* ctx, const uint8_t* id128, int rank, int world) { return qwgpu_comm_init_lane(ctx, 0, id128, rank, world); }
int qwgpu_comm_set_split_table(qwgpu_ctx* ctx, uint32_t n, const char* const* split_ids) {
  QW_API_BEGIN
  if (!ctx || !ctx->comm) qw::fail(QWGPU_EINVALID_ARG, "no communicator: call qwgpu_comm_init first");
  for (qw::Comm* c : ctx->lanes) if (c) qw::comm_set_split_table(c, n, split_ids);
  return 0;
  QW_API_END
}
void qwgpu_comm_destroy(qwgpu_ctx* ctx) {
  if (!ctx) return;
  for (qw::Comm*& c : ctx->lanes) { qw::comm_destroy(c); c = nullptr; }
  ctx->comm = nullptr;
}

// The host-staged exchange: this rank's LeafSearchResponse -> fixed-layout partial -> all ranks (only the used
// prefix travels: one 8-byte all-gather of the lengths, one of the longest prefix) -> merge_leaf_responses over
// the gathered partials. Carries everything a response holds (hits, aggregation bytes, failed_splits, stats).
static void exchange_responses(qw::Comm& comm, const qw::pb::SearchRequest& mreq, const uint8_t* mreq_pb, size_t mreq_len,
                               const uint8_t* local, size_t local_len, uint8_t** resp, size_t* resp_len) {
  const uint64_t stride = partial_bytes_for(mreq);
  std::vector<uint8_t> mine(stride);
  if (int rc = qwgpu_response_to_partial(mreq_pb, mreq_len, local, local_len, mine.data(), stride)) qw::fail(rc, "%s", qwgpu_last_error());
  uint64_t used = partial_used_bytes(mreq, mine.data());
  std::vector<uint64_t> lens((size_t)comm.world);
  qw::comm_allgather_host(&comm, (const uint8_t*)&used, (uint8_t*)lens.data(), 8);
  uint64_t longest = 0;
  for (uint64_t l : lens) longest = std::max(longest, l);
  if (longest > stride) qw::fail(QWGPU_EINTERNAL, "a rank announced a partial of %llu bytes (layout holds %llu)", (unsigned long long)longest, (unsigned long long)stride);
  longest = (longest + 15) & ~15ull;
  longest = std::min<uint64_t>(longest, stride);
  std::vector<uint8_t> packed(longest * (size_t)comm.world), gathered(stride * (size_t)comm.world);
  qw::comm_allgather_host(&comm, mine.data(), packed.data(), longest);
  for (int r = 0; r < comm.world; r++) memcpy(gathered.data() + (size_t)r * stride, packed.data() + (size_t)r * longest, longest);
  if (int rc = qwgpu_merge_partials(mreq_pb, mreq_len, (uint32_t)comm.world, gathered.data(), stride, resp, resp_len)) qw::fail(rc, "%s", qwgpu_last_error());
}

int qwgpu_leaf_search_allgather(qwgpu_ctx* ctx, const uint8_t* req, size_t req_len, uint8_t** resp, size_t* resp_len) {
  return qwgpu_leaf_search_allgather_lane(ctx, 0, req, req_len, resp, resp_len);
}

int qwgpu_leaf_search_allgather_lane(qwgpu_ctx* ctx, uint32_t lane, const uint8_t* req, size_t req_len, uint8_t** resp, size_t* resp_len) {
  QW_API_BEGIN
  qw::Engine& eng = engine_of(ctx);
  if (lane >= 16 || !ctx->lanes[lane]) qw::fail(QWGPU_EINVALID_ARG, "no communicator on lane %u: call qwgpu_comm_init_lane first", lane);
  qw::Comm& comm = *ctx->lanes[lane];
  qw::pb::LeafSearchRequest lr = qw::pb::decode_leaf_search_request(req, req_len);
  qw::pb::SearchRequest mreq = lr.search_request;
  mreq.max_hits += mreq.start_offset;
  mreq.start_offset = 0;
  const bool has_aggs = mreq.aggregation_request && !mreq.aggregation_request->empty();
  if (comm.world <= 1) return qwgpu_leaf_search(ctx, req, req_len, resp, resp_len);
  // every rank takes the same road: the request decides (hits without aggregations -> device-side exchange),
  // and after it the gathered counters do (a failed split anywhere -> the host-staged exchange carries the entries)
  bool staged = has_aggs || mreq.max_hits == 0;
  qw::pb::LeafSearchResponse m;
  if (!staged) {
  qw::LeafRun run;
  qw::run_leaf_raw(eng, lr, run, true, &comm);
  if (!run.gathered) qw::fail(QWGPU_EINTERNAL, "cross-rank merge did not run");
  uint64_t total_failed = 0;
  {
    for (const RankHeader& h : run.rank_headers) {
      m.num_hits += h.num_hits;
      m.num_attempted_splits += h.attempted;
      m.num_successful_splits += h.successful;
      total_failed += h.n_failed;
    }
    // the typed sort values come from the local splits' sort types
    if (run.which.empty() && !run.merged.empty()) qw::fail(QWGPU_EUNSUPPORTED, "a rank without searchable splits cannot type the merged sort values");
    const qw::SortTypes types = run.which.empty() ? qw::SortTypes{} : qw::sort_types(run.jobs, run.which);
    m.encoded_partial_hits.reserve(run.merged.size() * 72);
    for (const MergedHit& mh : run.merged) {
      if (mh.split >= comm.split_ids.size()) qw::fail(QWGPU_EINTERNAL, "gathered hit carries split rank %u (table has %zu)", mh.split, comm.split_ids.size());
      qw::append_hit(m.encoded_partial_hits, comm.split_ids[mh.split], mh.hit, types);
    }
  }
  staged = total_failed != 0;
  }
  if (!staged) {
    give(qw::pb::encode_leaf_search_response(m), resp, resp_len);
    return 0;
  }
  // host-staged road: this rank's complete response (a plain leaf search), exchanged and merged on every rank
  uint8_t* local = nullptr;
  size_t local_len = 0;
  if (qwgpu_leaf_search(ctx, req, req_len, &local, &local_len)) {
    // the other ranks are already waiting in the exchange: take part with a response that reports every split
    // of this rank as failed (the root retries them) instead of leaving the collective
    qw::pb::LeafSearchResponse err;
    const std::string why = qwgpu_last_error();
    for (auto& ref : lr.leaf_requests)
      for (auto& so : ref.split_offsets) { err.failed_splits.push_back({why, so.split_id, true}); err.num_attempted_splits++; }
    if (err.failed_splits.size() > 16) err.failed_splits.resize(16);  // (bounded tail; the counters still tell the whole story)
    give(qw::pb::encode_leaf_search_response(err), &local, &local_len);
  }
  struct Free { uint8_t* p; ~Free() { free(p); } } guard{local};
  const std::string mreq_pb = qw::pb::encode_search_request(mreq);
  exchange_responses(comm, mreq, (const uint8_t*)mreq_pb.data(), mreq_pb.size(), local, local_len, resp, resp_len);
  return 0;
  QW_API_END
}

int qwgpu_invoke_leaf_search(qwgpu_ctx* ctx, const uint8_t* req, size_t req_len, uint8_t** resp, size_t* resp_len) {
  QW_API_BEGIN
  qw::Engine& eng = engine_of(ctx);
  qw::pb::LeafSearchRequest lr = qw::pb::decode_leaf_search_request(req, req_len);
  give(qw::pb::encode_lambda_responses(qw::run_leaf(eng, lr)), resp, resp_len);
  return 0;
  QW_API_END
}

int qwgpu_compile_plan(const uint8_t* img, uint64_t img_len, const char* split_id, const uint8_t* search_request_pb,
                       size_t search_request_len, const char* doc_mapper_json, uint8_t** plan, size_t* plan_len) {
  QW_API_BEGIN
  qw::ImageView v;
  give(host_compile(v, img, img_len, split_id, search_request_pb, search_request_len, doc_mapper_json).bytes, plan, plan_len);
  return 0;
  QW_API_END
}

int qwgpu_build_leaf_response(const uint8_t* img, uint64_t img_len, const char* split_id, const uint8_t* search_request_pb,
                              size_t search_request_len, const char* doc_mapper_json, uint64_t num_hits, const QwHit* hits,
                              uint32_t num_partial_hits, const QwAggCell* cells, uint32_t num_cells, uint8_t** resp, size_t* resp_len) {
  QW_API_BEGIN
  qw::ImageView v;
  const qw::CompiledPlan cp = host_compile(v, img, img_len, split_id, search_request_pb, search_request_len, doc_mapper_json);
  qw::pb::LeafSearchResponse r = qw::build_split_response(cp, v, split_id ? split_id : "", num_hits, hits, num_partial_hits, cells, num_cells);
  give(qw::pb::encode_leaf_search_response(r), resp, resp_len);
  return 0;
  QW_API_END
}

int qwgpu_build_leaf_response_entries(const uint8_t* img, uint64_t img_len, const char* split_id, const uint8_t* search_request_pb,
                                      size_t search_request_len, const char* doc_mapper_json, uint64_t num_hits, const QwHit* hits,
                                      uint32_t num_partial_hits, const QwAggEntry* entries, uint32_t num_entries, uint8_t** resp, size_t* resp_len) {
  QW_API_BEGIN
  qw::ImageView v;
  const qw::CompiledPlan cp = host_compile(v, img, img_len, split_id, search_request_pb, search_request_len, doc_mapper_json);
  qw::pb::LeafSearchResponse r = qw::build_split_response(cp, v, split_id ? split_id : "", num_hits, hits, num_partial_hits, nullptr, 0,
                                                          entries, num_entries, true);
  give(qw::pb::encode_leaf_search_response(r), resp, resp_len);
  return 0;
  QW_API_END
}

int qwgpu_agg_layout(const uint8_t* img, uint64_t img_len, const char* split_id, const uint8_t* plan, size_t plan_len,
                     uint32_t* hashed, uint64_t* bound_cells) {
  QW_API_BEGIN
  qw::ImageView v;
  v.open(img, img_len);
  if (plan_len < sizeof(QwPlanHeader)) qw::fail(QWGPU_EINVALID_ARG, "plan too short");
  const QwPlanHeader* ph = (const QwPlanHeader*)plan;
  if (plan_len < sizeof(QwPlanHeader) + (size_t)ph->num_nodes * sizeof(QwPlanNode) + (size_t)ph->num_aggs * sizeof(QwAggNode))
    qw::fail(QWGPU_EINVALID_ARG, "plan truncated");
  const QwAggNode* aggs = (const QwAggNode*)(plan + sizeof(QwPlanHeader) + (size_t)ph->num_nodes * sizeof(QwPlanNode));
  for (uint32_t i = 0; i < ph->num_aggs; i++) {
    uint32_t depth = 0;
    for (uint32_t p = aggs[i].parent; p != 0xFFFFFFFFu; p = aggs[p].parent)
      if (p >= ph->num_aggs || ++depth > ph->num_aggs) qw::fail(QWGPU_EINVALID_ARG, "aggregation parent out of range");
  }
  *hashed = qw_agg_hashed(aggs, ph->num_aggs) ? 1u : 0u;
  *bound_cells = *hashed ? qw::agg_hashed_layout(aggs, ph->num_aggs, v, split_id ? split_id : "") : 0;
  return 0;
  QW_API_END
}

int qwgpu_regex_terms(const uint8_t* img, uint64_t img_len, const char* field, const char* regex, uint32_t** ords, uint64_t* num_ords,
                      uint64_t* transitions) {
  QW_API_BEGIN
  qw::ImageView v;
  v.open(img, img_len);
  const int f = v.find_field(field ? field : "");
  if (f < 0) qw::fail(QWGPU_EINVALID_ARG, "no text field `%s` in the split", field ? field : "");
  qw::rx::Regex re(regex ? regex : "");
  const std::vector<uint32_t> out = re.matching_terms(v, (uint32_t)f);
  *ords = nullptr;
  if (!out.empty()) {
    *ords = (uint32_t*)malloc(out.size() * 4);
    if (!*ords) qw::fail(QWGPU_EINTERNAL, "out of host memory");
    memcpy(*ords, out.data(), out.size() * 4);
  }
  *num_ords = out.size();
  *transitions = re.transitions();
  return 0;
  QW_API_END
}

int qwgpu_percentiles_table(const uint8_t* img, uint64_t img_len, uint32_t column, uint64_t** edges, uint64_t* num_bins,
                            int64_t* first_bin) {
  QW_API_BEGIN
  qw::ImageView v;
  v.open(img, img_len);
  if (column >= v.hdr->num_columns) qw::fail(QWGPU_EINVALID_ARG, "column %u (split has %u)", column, v.hdr->num_columns);
  const QwImgColumn& c = v.columns[column];
  if (c.type == QW_COL_STR || c.type == QW_COL_BYTES) qw::fail(QWGPU_EINVALID_AGG, "percentiles over a text or bytes column");
  if (c.type == QW_COL_IP) qw::fail(QWGPU_EUNSUPPORTED, "percentiles over an ip column are not supported on the GPU path");
  qw::dds::Table t;
  if (!qw::dds::column_table(c, true, &t)) qw::fail(QWGPU_EUNSUPPORTED, "percentiles over a column holding NaN or infinite values");
  *edges = nullptr;
  if (!t.edges.empty()) {
    *edges = (uint64_t*)malloc(t.edges.size() * 8);
    if (!*edges) qw::fail(QWGPU_EINTERNAL, "out of memory");
    memcpy(*edges, t.edges.data(), t.edges.size() * 8);
  }
  *num_bins = t.num_bins;
  *first_bin = t.ord_lo;
  return 0;
  QW_API_END
}

int qwgpu_merge_leaf_responses(const uint8_t* search_request_pb, size_t search_request_len, uint32_t n, const uint8_t* const* resps,
                               const size_t* resp_lens, uint8_t** merged, size_t* merged_len) {
  QW_API_BEGIN
  qw::pb::SearchRequest req = qw::pb::decode_search_request(qw::pb::Reader(search_request_pb, search_request_len));
  std::vector<qw::pb::LeafSearchResponse> parts;
  for (uint32_t i = 0; i < n; i++) parts.push_back(qw::pb::decode_leaf_search_response(resps[i], resp_lens[i]));
  qw::pb::LeafSearchResponse m;
  if (parts.empty()) {
    if (req.aggregation_request && !req.aggregation_request->empty())
      m.intermediate_aggregation_result = qw::merge_intermediate_aggs(qw::parse_agg_request(*req.aggregation_request), {});
  } else m = qw::merge_responses(req, std::move(parts));
  give(qw::pb::encode_leaf_search_response(m), merged, merged_len);
  return 0;
  QW_API_END
}

int qwgpu_finalize_aggregation(const char* aggregation_request_json, const uint8_t* intermediate, size_t intermediate_len, char** json_out) {
  QW_API_BEGIN
  std::vector<qw::AggReq> reqs = qw::parse_agg_request(aggregation_request_json ? aggregation_request_json : "{}");
  std::string js = qw::finalize_aggs_json(reqs, std::string((const char*)intermediate, intermediate_len));
  *json_out = (char*)malloc(js.size() + 1);
  if (!*json_out) qw::fail(QWGPU_EINTERNAL, "out of memory");
  memcpy(*json_out, js.c_str(), js.size() + 1);
  return 0;
  QW_API_END
}

int qwgpu_partial_size(const uint8_t* search_request_pb, size_t search_request_len, uint64_t* partial_bytes) {
  QW_API_BEGIN
  *partial_bytes = partial_bytes_for(qw::pb::decode_search_request(qw::pb::Reader(search_request_pb, search_request_len)));
  return 0;
  QW_API_END
}

int qwgpu_response_to_partial(const uint8_t* search_request_pb, size_t search_request_len, const uint8_t* resp, size_t resp_len,
                              uint8_t* partial, uint64_t partial_bytes) {
  QW_API_BEGIN
  qw::pb::SearchRequest req = qw::pb::decode_search_request(qw::pb::Reader(search_request_pb, search_request_len));
  if (partial_bytes != partial_bytes_for(req)) qw::fail(QWGPU_EINVALID_ARG, "partial buffer size mismatch");
  qw::pb::LeafSearchResponse r = qw::pb::decode_leaf_search_response(resp, resp_len);
  size_t k = (size_t)(req.max_hits + req.start_offset);
  if (r.partial_hits.size() > k) qw::fail(QWGPU_EINVALID_ARG, "response holds more hits than max_hits + start_offset");
  memset(partial, 0, partial_bytes);
  uint64_t hdr[4] = {kPartMagic, r.num_hits, r.num_attempted_splits, r.num_successful_splits};
  memcpy(partial, hdr, 32);
  uint32_t meta[4] = {(uint32_t)r.partial_hits.size(), 0, (uint32_t)r.failed_splits.size(), 0};
  uint8_t* p = partial + 48;
  for (auto& h : r.partial_hits) {
    if (h.split_id.size() > 40) qw::fail(QWGPU_EUNSUPPORTED, "split ids longer than 40 bytes do not fit the fixed-size partial");
    auto pack = [](bool has, const qw::pb::SortValue& v, uint64_t* out) -> uint8_t {
      if (!has) return 0xFF;
      switch (v.kind) {
        case qw::pb::SortValue::U64: *out = v.u; break;
        case qw::pb::SortValue::I64: *out = (uint64_t)v.i; break;
        case qw::pb::SortValue::F64: memcpy(out, &v.f, 8); break;
        case qw::pb::SortValue::Bool: *out = v.b; break;
        default: *out = 0;
      }
      return (uint8_t)v.kind;
    };
    uint64_t v1 = 0, v2 = 0;
    p[0] = pack(h.has_sv1, h.sv1, &v1);
    p[1] = pack(h.has_sv2, h.sv2, &v2);
    uint16_t sl = (uint16_t)h.split_id.size();
    memcpy(p + 2, &sl, 2);
    memcpy(p + 4, &h.doc_id, 4);
    memcpy(p + 8, &v1, 8);
    memcpy(p + 16, &v2, 8);
    memcpy(p + 24, h.split_id.data(), sl);
    p += kHitBytes;
  }
  if (r.intermediate_aggregation_result) {
    if (r.intermediate_aggregation_result->size() > kAggCap) qw::fail(QWGPU_EUNSUPPORTED, "intermediate aggregation result exceeds the fixed partial capacity");
    meta[1] = (uint32_t)r.intermediate_aggregation_result->size();
    memcpy(partial + 48 + k * kHitBytes + kTailCap, r.intermediate_aggregation_result->data(), meta[1]);
  }
  // tail: what the root needs besides hits and buckets — the failed_splits entries (its retry is keyed on them)
  // and the resource statistics — as a LeafSearchResponse message holding only those fields
  if (!r.failed_splits.empty() || r.resource_stats) {
    qw::pb::LeafSearchResponse t;
    t.failed_splits = r.failed_splits;
    t.resource_stats = r.resource_stats;
    const std::string tail = qw::pb::encode_leaf_search_response(t);
    if (tail.size() > kTailCap) qw::fail(QWGPU_EUNSUPPORTED, "%zu failed splits do not fit the fixed-size partial (%zu bytes)", r.failed_splits.size(), (size_t)kTailCap);
    meta[3] = (uint32_t)tail.size();
    memcpy(partial + 48 + k * kHitBytes, tail.data(), tail.size());
  }
  memcpy(partial + 32, meta, 16);
  return 0;
  QW_API_END
}

int qwgpu_merge_partials(const uint8_t* search_request_pb, size_t search_request_len, uint32_t n_ranks, const uint8_t* gathered,
                         uint64_t partial_bytes, uint8_t** merged, size_t* merged_len) {
  QW_API_BEGIN
  qw::pb::SearchRequest req = qw::pb::decode_search_request(qw::pb::Reader(search_request_pb, search_request_len));
  if (partial_bytes != partial_bytes_for(req)) qw::fail(QWGPU_EINVALID_ARG, "partial buffer size mismatch");
  size_t k = (size_t)(req.max_hits + req.start_offset);
  std::vector<qw::pb::LeafSearchResponse> parts;
  for (uint32_t r = 0; r < n_ranks; r++) {
    const uint8_t* base = gathered + (size_t)r * partial_bytes;
    uint64_t hdr[4];
    uint32_t meta[4];
    memcpy(hdr, base, 32);
    memcpy(meta, base + 32, 16);
    if (hdr[0] != kPartMagic) qw::fail(QWGPU_EINVALID_ARG, "rank %u partial has a bad header", r);
    // the gathered bytes come from other processes: nothing in them is trusted
    if (meta[0] > k) qw::fail(QWGPU_EINVALID_ARG, "rank %u partial claims %u hits (max %zu)", r, meta[0], k);
    if (meta[1] > kAggCap || 48 + k * kHitBytes + kTailCap + (size_t)meta[1] > partial_bytes) qw::fail(QWGPU_EINVALID_ARG, "rank %u partial claims %u aggregation bytes", r, meta[1]);
    if (meta[3] > kTailCap) qw::fail(QWGPU_EINVALID_ARG, "rank %u partial claims a tail of %u bytes", r, meta[3]);
    qw::pb::LeafSearchResponse lr;
    lr.num_hits = hdr[1];
    lr.num_attempted_splits = hdr[2];
    lr.num_successful_splits = hdr[3];
    const uint8_t* p = base + 48;
    for (uint32_t i = 0; i < meta[0]; i++, p += kHitBytes) {
      qw::pb::PartialHit h;
      auto unpack = [](uint8_t kind, uint64_t v, bool* has, qw::pb::SortValue* out) {
        if (kind == 0xFF) { *has = false; return; }
        *has = true;
        out->kind = (qw::pb::SortValue::Kind)kind;
        switch (out->kind) {
          case qw::pb::SortValue::U64: out->u = v; break;
          case qw::pb::SortValue::I64: out->i = (int64_t)v; break;
          case qw::pb::SortValue::F64: memcpy(&out->f, &v, 8); break;
          case qw::pb::SortValue::Bool: out->b = v != 0; break;
          default: break;
        }
      };
      uint64_t v1, v2;
      uint16_t sl;
      memcpy(&sl, p + 2, 2);
      memcpy(&h.doc_id, p + 4, 4);
      memcpy(&v1, p + 8, 8);
      memcpy(&v2, p + 16, 8);
      unpack(p[0], v1, &h.has_sv1, &h.sv1);
      unpack(p[1], v2, &h.has_sv2, &h.sv2);
      if (sl > 40) qw::fail(QWGPU_EINVALID_ARG, "rank %u partial holds a split id of %u bytes", r, (unsigned)sl);
      h.split_id.assign((const char*)p + 24, sl);
      lr.partial_hits.push_back(std::move(h));
    }
    if (meta[1]) lr.intermediate_aggregation_result = std::string((const char*)base + 48 + k * kHitBytes + kTailCap, meta[1]);
    if (meta[3]) {
      qw::pb::LeafSearchResponse t = qw::pb::decode_leaf_search_response(base + 48 + k * kHitBytes, meta[3]);
      lr.failed_splits = std::move(t.failed_splits);
      lr.resource_stats = t.resource_stats;
    }
    if (lr.failed_splits.size() != meta[2]) qw::fail(QWGPU_EINVALID_ARG, "rank %u partial reports %u failed splits but carries %zu", r, meta[2], lr.failed_splits.size());
    parts.push_back(std::move(lr));
  }
  qw::pb::LeafSearchResponse m = qw::merge_responses(req, std::move(parts));
  give(qw::pb::encode_leaf_search_response(m), merged, merged_len);
  return 0;
  QW_API_END
}

}  // extern "C"
