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
#include <algorithm>
#include <chrono>
#include <tuple>

#include "compile.h"
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
                                            const QwAggCell* cells, size_t ncells) {
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
  if (cp.header.num_aggs) r.intermediate_aggregation_result = build_intermediate_aggs(cp, img, cells, ncells);
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
};

struct LeafRun {
  std::vector<SplitJob> jobs;
  std::vector<size_t> which;      // jobs[which[k]] <-> outs[k]
  std::vector<SplitOutput> outs;
  BatchStats st;
  uint64_t wall_us = 0;
  bool merged_valid = false;       // the engine merged the per-split top-K lists on the device
  std::vector<MergedHit> merged;   // best-first; .split = index into `jobs` (gathered: global split rank)
  bool gathered = false;           // `merged` is the cross-rank result; rank_headers[r] = rank r's counters
  std::vector<RankHeader> rank_headers;
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
static void sort_orders(const pb::SearchRequest& r, int* o1, int* o2);

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

static void run_leaf_raw(Engine& eng, const pb::LeafSearchRequest& lr, LeafRun& run, bool want_merged = false, const Comm* comm = nullptr) {
  using clock = std::chrono::steady_clock;
  const pb::SearchRequest& sreq = lr.search_request;
  const auto t_compile = clock::now();
  Json ast = parse_json(sreq.query_ast, QWGPU_EINVALID_QUERY);  // once per request
  for (auto& ref : lr.leaf_requests) {
    if (ref.doc_mapper_ord >= lr.doc_mappers.size()) fail(QWGPU_EINVALID_ARG, "Internal error: doc_mapper_ord out of bounds");
    DocMapperInfo dm = parse_doc_mapper(lr.doc_mappers[ref.doc_mapper_ord]);
    // per-split request rewrite (a16); the jobs keep the request's split order (the processing order of a
    // batch is not observable). Across ranks every split goes to the device: the counters of the exchanged
    // record are built there.
    std::vector<SplitRequest> opt = optimize_split_requests(sreq, ast, dm.timestamp_field, ref.split_offsets);
    std::vector<const SplitRequest*> by_pos(ref.split_offsets.size(), nullptr);
    for (const SplitRequest& q : opt) by_pos[q.input_pos] = &q;
    static const bool no_prune = getenv("QWGPU_NO_PRUNING") != nullptr;
    pb::SearchRequest count_req;
    bool have_count_req = false;
    for (size_t si = 0; si < ref.split_offsets.size(); si++) {
      const pb::SplitIdAndFooterOffsets& so = ref.split_offsets[si];
      const SplitRequest& q = *by_pos[si];
      if (q.skipped && !comm && !no_prune) continue;  // (PrunedBeforeWarmup: contributes nothing, not even to the split counters)
      SplitJob j;
      j.meta = so;
      if (q.metadata_count && !comm && !no_prune) {
        j.metadata_count = true;
        run.jobs.push_back(std::move(j));
        continue;
      }
      const pb::SearchRequest* req = &sreq;
      if (q.hits_disabled && !no_prune) {
        if (!have_count_req) { count_req = sreq; disable_search_request_hits(count_req); have_count_req = true; }
        req = &count_req;
      }
      j.dev = eng.find(so.split_id);
      try {
        if (!j.dev) fail(QWGPU_ENOTFOUND, "split `%s` is not resident on this GPU", so.split_id.c_str());
        j.plan = compile_plan(j.dev->view, so.split_id, *req, dm, &so, &ast);
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
    if (!run.jobs[i].error_code && !run.jobs[i].metadata_count) {
      devs.push_back(run.jobs[i].dev);
      plans.push_back((const uint8_t*)run.jobs[i].plan.bytes.data());
      lens.push_back(run.jobs[i].plan.bytes.size());
      run.which.push_back(i);
    }
  auto t0 = clock::now();
  if (getenv("QWGPU_TRACE"))
    fprintf(stderr, "[qwgpu] compile: %ld us for %zu splits\n", (long)std::chrono::duration_cast<std::chrono::microseconds>(t0 - t_compile).count(), run.jobs.size());
  static const bool host_merge = getenv("QWGPU_HOST_MERGE") != nullptr;
  MergeSpec ms;
  GatherSpec gs;
  const bool gathering = comm && comm->world > 1 && sreq.max_hits + sreq.start_offset > 0;
  if (gathering && !same_sort_types(run.jobs, run.which)) fail(QWGPU_EUNSUPPORTED, "the splits of this rank disagree on the sort field types: cross-rank merge on the device is not possible");
  if ((gathering || (want_merged && !host_merge && devs.size() > 1)) && sreq.max_hits + sreq.start_offset > 0 && same_sort_types(run.jobs, run.which)) {
    int o1, o2;
    sort_orders(sreq, &o1, &o2);
    ms.k = (uint32_t)(sreq.max_hits + sreq.start_offset);
    ms.order1 = (uint32_t)o1; ms.order2 = (uint32_t)o2;
    const size_t n = run.which.size();
    std::vector<size_t> by_id(n);
    for (size_t i = 0; i < n; i++) by_id[i] = i;
    std::sort(by_id.begin(), by_id.end(), [&](size_t a, size_t b) { return run.jobs[run.which[a]].meta.split_id < run.jobs[run.which[b]].meta.split_id; });
    ms.rank.resize(n);
    for (size_t r = 0; r < n; r++) ms.rank[by_id[r]] = (uint32_t)r;
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
  for (size_t k = 0; k < run.which.size(); k++) {
    size_t i = run.which[k];
    SplitOutput& o = run.outs[k];
    if (o.status) { results[i].is_error = true; results[i].error = o.error; continue; }
    pb::LeafSearchResponse r = build_split_response(run.jobs[i].plan, run.jobs[i].dev->view, run.jobs[i].meta.split_id, o.num_hits,
                                                    o.hits.data(), o.hits.size(), o.cells.data(), o.cells.size());
    r.resource_stats = split_stats(run, k);
    results[i].response = std::move(r);
  }
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
  // rank of every split id (tie-break uses the split id string order)
  std::vector<size_t> by_id(n);
  for (size_t i = 0; i < n; i++) by_id[i] = i;
  std::sort(by_id.begin(), by_id.end(), [&](size_t a, size_t b) { return run.jobs[run.which[a]].meta.split_id < run.jobs[run.which[b]].meta.split_id; });
  std::vector<uint32_t> rank(n);
  for (size_t r = 0; r < n; r++) rank[by_id[r]] = (uint32_t)r;
  const CompiledPlan& p0 = run.jobs[run.which[0]].plan;
  // sort-field type of each key: taken from a split that actually has the column (splits without it
  // only produce None values)
  int sft[2] = {p0.sort_field_type[0], p0.sort_field_type[1]};
  for (int i = 0; i < 2; i++)
    for (size_t s2 = 0; s2 < n; s2++) {
      const CompiledPlan& pp = run.jobs[run.which[s2]].plan;
      if (pp.header.sort[i].kind == QW_SORT_COLUMN && pp.header.sort[i].column != 0xFFFFFFFFu) { sft[i] = pp.sort_field_type[i]; break; }
    }
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
    const uint64_t t = ((uint64_t)rank[sidx] << 32) | h.doc_id;
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
    if (j.plan.header.num_aggs) agg_parts.push_back({&j.plan, &j.dev->view, o.cells.data(), o.cells.size()});
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
      const QwHit& h = mh.hit;
      pb::SortValue sv1, sv2;
      if (h.flags & 1) sv1 = typed_sort_value(p0.header.sort[0].kind, sft[0], h.v1);
      if (h.flags & 2) sv2 = typed_sort_value(p0.header.sort[1].kind, sft[1], h.v2);
      pb::append_partial_hit(m.encoded_partial_hits, 2, run.jobs[mh.split].meta.split_id, 0, h.doc_id, (h.flags & 1) != 0, sv1, (h.flags & 2) != 0, sv2);
      taken++;
    }
    heap.clear();
  }
  while (!heap.empty() && taken < k) {
    std::pop_heap(heap.begin(), heap.end());
    size_t s = heap.back().s;
    const SplitJob& j = run.jobs[run.which[s]];
    const QwHit& h = run.outs[s].hits[pos[s]];
    pb::SortValue sv1, sv2;
    if (h.flags & 1) sv1 = typed_sort_value(p0.header.sort[0].kind, sft[0], h.v1);
    if (h.flags & 2) sv2 = typed_sort_value(p0.header.sort[1].kind, sft[1], h.v2);
    pb::append_partial_hit(m.encoded_partial_hits, 2, j.meta.split_id, 0, h.doc_id, (h.flags & 1) != 0, sv1, (h.flags & 2) != 0, sv2);
    taken++;
    if (++pos[s] < run.outs[s].hits.size()) { heap.back() = head_of(s, run.outs[s].hits[pos[s]]); std::push_heap(heap.begin(), heap.end()); }
    else heap.pop_back();
  }
  if (sreq.aggregation_request && !sreq.aggregation_request->empty())
    m.intermediate_aggregation_result = build_and_merge_intermediate_aggs(p0.agg_request, agg_parts);
  if (any_stats) m.resource_stats = stats_acc;
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
  if (run.which.empty()) {
    if (mreq.aggregation_request && !mreq.aggregation_request->empty())
      merged.intermediate_aggregation_result = qw::merge_intermediate_aggs(qw::parse_agg_request(*mreq.aggregation_request), {});
  } else if (same_types) {
    merged = qw::leaf_merge_fast(mreq, run);
  } else {
    std::vector<qw::pb::LeafSearchResponse> parts;
    for (size_t k = 0; k < run.which.size(); k++) {
      const qw::SplitJob& j = run.jobs[run.which[k]];
      qw::SplitOutput& o = run.outs[k];
      qw::pb::LeafSearchResponse r = qw::build_split_response(j.plan, j.dev->view, j.meta.split_id, o.num_hits, o.hits.data(), o.hits.size(), o.cells.data(), o.cells.size());
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
    fprintf(stderr, "[qwgpu] leaf_search: decode %ld us, compile+search %ld us (engine wall %lu us, device %.0f us, %u launches), merge %ld us, encode %ld us\n",
            us(t_start, t_dec), us(t_dec, t_run), (unsigned long)run.wall_us, run.st.gpu_time_us, run.st.launches, us(t_run, t_merge), us(t_merge, tclock::now()));
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
    for (const qw::RankHeader& h : run.rank_headers) {
      m.num_hits += h.num_hits;
      m.num_attempted_splits += h.attempted;
      m.num_successful_splits += h.successful;
      total_failed += h.n_failed;
    }
    // sort-field types for the typed sort values: from a local split that has the column
    const qw::CompiledPlan* p0 = run.which.empty() ? nullptr : &run.jobs[run.which[0]].plan;
    if (!p0 && !run.merged.empty()) qw::fail(QWGPU_EUNSUPPORTED, "a rank without searchable splits cannot type the merged sort values");
    int sft[2] = {0, 0};
    if (p0) {
      sft[0] = p0->sort_field_type[0]; sft[1] = p0->sort_field_type[1];
      for (int i = 0; i < 2; i++)
        for (size_t s2 = 0; s2 < run.which.size(); s2++) {
          const qw::CompiledPlan& pp = run.jobs[run.which[s2]].plan;
          if (pp.header.sort[i].kind == QW_SORT_COLUMN && pp.header.sort[i].column != 0xFFFFFFFFu) { sft[i] = pp.sort_field_type[i]; break; }
        }
    }
    m.encoded_partial_hits.reserve(run.merged.size() * 72);
    for (const qw::MergedHit& mh : run.merged) {
      if (mh.split >= comm.split_ids.size()) qw::fail(QWGPU_EINTERNAL, "gathered hit carries split rank %u (table has %zu)", mh.split, comm.split_ids.size());
      const QwHit& h = mh.hit;
      qw::pb::SortValue sv1, sv2;
      if (h.flags & 1) sv1 = qw::typed_sort_value(p0->header.sort[0].kind, sft[0], h.v1);
      if (h.flags & 2) sv2 = qw::typed_sort_value(p0->header.sort[1].kind, sft[1], h.v2);
      qw::pb::append_partial_hit(m.encoded_partial_hits, 2, comm.split_ids[mh.split], 0, h.doc_id, (h.flags & 1) != 0, sv1, (h.flags & 2) != 0, sv2);
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
  v.open(img, img_len);
  qw::pb::SearchRequest req = qw::pb::decode_search_request(qw::pb::Reader(search_request_pb, search_request_len));
  qw::DocMapperInfo dm = qw::parse_doc_mapper(doc_mapper_json ? doc_mapper_json : "");
  qw::CompiledPlan cp = qw::compile_plan(v, split_id ? split_id : "", req, dm, nullptr);
  give(cp.bytes, plan, plan_len);
  return 0;
  QW_API_END
}

int qwgpu_build_leaf_response(const uint8_t* img, uint64_t img_len, const char* split_id, const uint8_t* search_request_pb,
                              size_t search_request_len, const char* doc_mapper_json, uint64_t num_hits, const QwHit* hits,
                              uint32_t num_partial_hits, const QwAggCell* cells, uint32_t num_cells, uint8_t** resp, size_t* resp_len) {
  QW_API_BEGIN
  qw::ImageView v;
  v.open(img, img_len);
  qw::pb::SearchRequest req = qw::pb::decode_search_request(qw::pb::Reader(search_request_pb, search_request_len));
  qw::DocMapperInfo dm = qw::parse_doc_mapper(doc_mapper_json ? doc_mapper_json : "");
  qw::CompiledPlan cp = qw::compile_plan(v, split_id ? split_id : "", req, dm, nullptr);
  qw::pb::LeafSearchResponse r = qw::build_split_response(cp, v, split_id ? split_id : "", num_hits, hits, num_partial_hits, cells, num_cells);
  give(qw::pb::encode_leaf_search_response(r), resp, resp_len);
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
