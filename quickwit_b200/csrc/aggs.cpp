// aggs.cpp — aggregation request parsing, lowering to dense GPU bucket spaces, intermediate
// results (build / merge / serialise) and finalisation.
//
// Reference behaviour restated (the engine itself is tantivy::aggregation, external):
//   * request shape + parameters: docs/reference/aggregation.md:40-700
//   * leaf: AggregationSegmentCollector::harvest -> IntermediateAggregationResults, cut to
//     `segment_size` per split with sum_other_doc_count / doc_count_error_upper_bound
//     (quickwit-search/src/collector.rs:577-581; aggregation.md:500-560)
//   * merge: IntermediateAggregationResults::merge_fruits (collector.rs:870-911)
//   * final: into_final_result (quickwit-search/src/root.rs:1105-1135): buckets cut to `size`,
//     histogram gaps filled when min_doc_count == 0, extended_bounds, key_as_string.
#include <algorithm>
#include <cerrno>
#include <cmath>
#include <map>
#include <set>
#include <tuple>
#include <memory>

#include "compile.h"
#include "ddsketch.h"
#include "device_types.h"
#include "ip_addr.h"

namespace qw {

// ---- request parsing -----------------------------------------------------------------------------------
static double parse_duration_ms(const std::string& s, bool allow_negative) {
  // fixed_interval / offset syntax: <int><unit>, unit in ms|s|m|h|d (aggregation.md:300-320)
  size_t i = 0;
  bool neg = false;
  if (i < s.size() && (s[i] == '-' || s[i] == '+')) { neg = s[i] == '-'; i++; }
  if (neg && !allow_negative) fail(QWGPU_EINVALID_AGG, "negative duration `%s`", s.c_str());
  size_t j = i;
  while (j < s.size() && isdigit((unsigned char)s[j])) j++;
  if (j == i) fail(QWGPU_EINVALID_AGG, "invalid duration `%s`", s.c_str());
  double n = strtod(s.substr(i, j - i).c_str(), nullptr);
  std::string unit = s.substr(j);
  double mult;
  if (unit == "ms") mult = 1;
  else if (unit == "s") mult = 1000;
  else if (unit == "m") mult = 60000;
  else if (unit == "h") mult = 3600000;
  else if (unit == "d") mult = 86400000;
  else fail(QWGPU_EINVALID_AGG, "unsupported duration unit in `%s` (only fixed intervals ms|s|m|h|d)", s.c_str());
  return (neg ? -1 : 1) * n * mult;
}

static double num_or(const Json& j, const char* k, double d) {
  const Json* v = j.get(k);
  if (!v) return d;
  if (v->is_num()) return v->as_f64();
  if (v->is_str()) return strtod(v->s.c_str(), nullptr);
  return d;
}

// `after` value of a composite source: type-tagged strings ("str:…", "i64:…", "u64:…", "f64:…", "bool:…", the form
// after_key is written in) or plain JSON strings, numbers, booleans and null
static CompKey parse_after_value(const Json& v, const std::string& src) {
  CompKey k;
  auto bad = [&]() { fail(QWGPU_EINVALID_AGG, "composite `after` value of source `%s` is not a valid key", src.c_str()); };
  switch (v.type) {
    case Json::Null: k.t = CompKey::Null; return k;
    case Json::Bool: k.t = CompKey::Bool; k.u = v.b ? 1 : 0; return k;
    case Json::U64: k.t = CompKey::U64; k.u = v.u; return k;
    case Json::I64: k.t = CompKey::I64; k.i = v.i; return k;
    case Json::F64: k.t = CompKey::F64; k.f = v.f; return k;
    case Json::Str: break;
    default: bad();
  }
  const std::string& s = v.s;
  const size_t colon = s.find(':');
  const std::string tag = colon == std::string::npos ? "" : s.substr(0, colon), rest = colon == std::string::npos ? "" : s.substr(colon + 1);
  char* end = nullptr;
  errno = 0;
  if (tag == "str") { k.t = CompKey::Str; k.s = rest; }
  else if (tag == "i64") { k.t = CompKey::I64; k.i = strtoll(rest.c_str(), &end, 10); if (rest.empty() || *end || errno) bad(); }
  else if (tag == "u64") { k.t = CompKey::U64; k.u = strtoull(rest.c_str(), &end, 10); if (rest.empty() || rest[0] == '-' || *end || errno) bad(); }
  else if (tag == "f64") { k.t = CompKey::F64; k.f = strtod(rest.c_str(), &end); if (rest.empty() || *end) bad(); }
  else if (tag == "bool") { k.t = CompKey::Bool; if (rest != "true" && rest != "false") bad(); k.u = rest == "true"; }
  else { k.t = CompKey::Str; k.s = s; }
  return k;
}

// composite: {"size": n, "sources": [{name: {terms | histogram | date_histogram: {...}}}, ...], "after": {...}}
static void parse_composite(const Json& spec, AggReq& a, int depth) {
  if (depth > 0) fail(QWGPU_EUNSUPPORTED, "composite aggregation `%s` below another aggregation is not implemented on the GPU path", a.name.c_str());
  if (!spec.is_obj()) fail(QWGPU_EINVALID_AGG, "composite aggregation `%s` must be a JSON object", a.name.c_str());
  a.kind = AggReq::Composite;
  const double size = num_or(spec, "size", 10);
  if (!(size >= 1) || size != std::floor(size)) fail(QWGPU_EINVALID_AGG, "composite `size` must be a positive integer");
  if (size > QW_AGG_COMP_MAX_SIZE) fail(QWGPU_EUNSUPPORTED, "composite `size` %g exceeds the bucket limit %u", size, QW_AGG_COMP_MAX_SIZE);
  a.size = (uint32_t)size;
  const Json* srcs = spec.get("sources");
  if (!srcs || !srcs->is_arr() || srcs->arr.empty()) fail(QWGPU_EINVALID_AGG, "composite aggregation `%s` requires a non-empty `sources` list", a.name.c_str());
  for (const Json& e : srcs->arr) {
    if (!e.is_obj() || e.obj.size() != 1 || !e.obj[0].second.is_obj() || e.obj[0].second.obj.size() != 1)
      fail(QWGPU_EINVALID_AGG, "a composite source must be an object {name: {type: {...}}}");
    AggReq s;
    s.name = e.obj[0].first;
    for (const AggReq& o : a.sources) if (o.name == s.name) fail(QWGPU_EINVALID_AGG, "duplicate composite source name `%s`", s.name.c_str());
    const std::string& t = e.obj[0].second.obj[0].first;
    const Json& p = e.obj[0].second.obj[0].second;
    if (!p.is_obj()) fail(QWGPU_EINVALID_AGG, "composite source `%s` must be a JSON object", s.name.c_str());
    for (const char* k : {"missing_order", "format", "script", "calendar_interval", "time_zone"})
      if (p.get(k)) fail(QWGPU_EUNSUPPORTED, "`%s` of composite source `%s` is not implemented on the GPU path", k, s.name.c_str());
    const Json* f = p.get("field");
    if (!f || !f->is_str()) fail(QWGPU_EINVALID_AGG, "composite source `%s` requires a `field`", s.name.c_str());
    s.field = f->s;
    if (t == "terms") s.kind = AggReq::Terms;
    else if (t == "histogram") {
      s.kind = AggReq::Histogram;
      s.interval = num_or(p, "interval", 0);
      s.offset = num_or(p, "offset", 0);
    } else if (t == "date_histogram") {
      s.kind = AggReq::DateHistogram;
      const Json* fi = p.get("fixed_interval");
      if (p.get("interval") || !fi || !fi->is_str()) fail(QWGPU_EINVALID_AGG, "composite date_histogram source `%s` requires `fixed_interval`", s.name.c_str());
      s.interval = parse_duration_ms(fi->s, false);
      if (const Json* off = p.get("offset")) s.offset = off->is_str() ? parse_duration_ms(off->s, true) : off->as_f64();
    } else fail(QWGPU_EINVALID_AGG, "unknown composite source type `%s`", t.c_str());
    if (s.kind != AggReq::Terms && !(s.interval > 0)) fail(QWGPU_EINVALID_AGG, "histogram interval must be larger than 0");
    s.order_desc = false;
    if (const Json* o = p.get("order")) {
      if (!o->is_str() || (o->s != "asc" && o->s != "desc")) fail(QWGPU_EINVALID_AGG, "composite source `%s`: `order` must be \"asc\" or \"desc\"", s.name.c_str());
      s.order_desc = o->s == "desc";
    }
    s.has_missing = p.bool_or("missing_bucket", false);
    a.sources.push_back(std::move(s));
  }
  if (const Json* af = spec.get("after")) {
    if (!af->is_obj()) fail(QWGPU_EINVALID_AGG, "composite `after` must be an object");
    a.has_after = true;
    a.after.resize(a.sources.size());
    std::vector<bool> seen(a.sources.size(), false);
    for (auto& kv : af->obj) {
      size_t i = 0;
      while (i < a.sources.size() && a.sources[i].name != kv.first) i++;
      if (i == a.sources.size()) fail(QWGPU_EINVALID_AGG, "composite `after` names `%s`, which is not a source", kv.first.c_str());
      if (seen[i]) fail(QWGPU_EINVALID_AGG, "composite `after` names `%s` twice", kv.first.c_str());
      seen[i] = true;
      const AggReq& s = a.sources[i];
      CompKey k = parse_after_value(kv.second, s.name);
      if (k.t == CompKey::Null && !s.has_missing) fail(QWGPU_EINVALID_AGG, "composite `after` is null for source `%s`, which has no missing_bucket", s.name.c_str());
      if (s.kind != AggReq::Terms && k.t != CompKey::Null && !k.numeric())
        fail(QWGPU_EINVALID_AGG, "composite `after` value of histogram source `%s` must be a number", s.name.c_str());
      a.after[i] = std::move(k);
    }
    for (size_t i = 0; i < seen.size(); i++)
      if (!seen[i]) fail(QWGPU_EINVALID_AGG, "composite `after` lacks source `%s`", a.sources[i].name.c_str());
  }
}

// `missing` of a metric aggregation (percentiles and the stats family): a JSON number, taken as an f64
static void parse_metric_missing(const Json& spec, AggReq& a, const char* type) {
  if (const Json* m = spec.get("missing")) {
    if (!m->is_num()) fail(QWGPU_EINVALID_AGG, "%s `missing` must be a number", type);
    a.has_missing = true;
    a.missing = *m;
  }
}

// percentiles: {"field", "percents": [..] (default 1, 5, 25, 50, 75, 95, 99), "keyed" (default true), "missing": number}
static void parse_percentiles(const Json& spec, AggReq& a) {
  a.kind = AggReq::Percentiles;
  if (a.field.empty()) fail(QWGPU_EINVALID_AGG, "percentiles aggregation `%s` requires a `field`", a.name.c_str());
  a.percents = {1, 5, 25, 50, 75, 95, 99};
  if (const Json* p = spec.get("percents")) {
    if (!p->is_arr()) fail(QWGPU_EINVALID_AGG, "percentiles `percents` must be a list of numbers");
    a.percents.clear();
    for (const Json& x : p->arr) {
      if (!x.is_num()) fail(QWGPU_EINVALID_AGG, "percentiles `percents` must be a list of numbers");
      const double v = x.as_f64();
      if (!(v >= 0 && v <= 100)) fail(QWGPU_EINVALID_AGG, "percent %g is not between 0 and 100", v);
      a.percents.push_back(v);
    }
  }
  a.keyed = spec.bool_or("keyed", true);
  parse_metric_missing(spec, a, "percentiles");
}

static void parse_agg_map(const Json& j, std::vector<AggReq>& out, int depth) {
  if (!j.is_obj()) fail(QWGPU_EINVALID_AGG, "aggregation request must be a JSON object");
  if (depth > 8) fail(QWGPU_EINVALID_AGG, "aggregation nesting too deep");
  for (auto& kv : j.obj) {
    AggReq a;
    a.name = kv.first;
    const Json& body = kv.second;
    bool found = false;
    for (auto& p : body.obj) {
      const std::string& t = p.first;
      const Json& spec = p.second;
      if (t == "aggs" || t == "aggregations") { parse_agg_map(spec, a.children, depth + 1); continue; }
      if (found) fail(QWGPU_EINVALID_AGG, "aggregation `%s` has more than one type", a.name.c_str());
      found = true;
      a.field = spec.str_or("field", "");
      if (t == "composite") parse_composite(spec, a, depth);
      else if (t == "terms") {
        a.kind = AggReq::Terms;
        a.size = (uint32_t)num_or(spec, "size", 10);
        double ss = -1;
        for (const char* k : {"split_size", "segment_size", "shard_size"}) if (spec.get(k)) ss = num_or(spec, k, -1);
        a.segment_size = ss >= 0 ? (uint32_t)ss : a.size * 10;
        a.segment_size = std::max(a.segment_size, a.size);
        a.min_doc_count = (uint64_t)num_or(spec, "min_doc_count", 1);
        if (const Json* m = spec.get("missing")) { a.has_missing = true; a.missing = *m; }
        if (const Json* o = spec.get("order")) {
          if (!o->is_obj() || o->obj.size() != 1) fail(QWGPU_EINVALID_AGG, "terms `order` must be an object with one property");
          a.order_target = o->obj[0].first;
          a.order_desc = o->obj[0].second.is_str() && o->obj[0].second.s == "desc";
        }
      } else if (t == "histogram" || t == "date_histogram") {
        a.kind = t == "histogram" ? AggReq::Histogram : AggReq::DateHistogram;
        if (a.kind == AggReq::DateHistogram) {
          if (spec.get("interval") || spec.get("calendar_interval")) fail(QWGPU_EINVALID_AGG, "date_histogram only supports `fixed_interval`");
          const Json* fi = spec.get("fixed_interval");
          if (!fi || !fi->is_str()) fail(QWGPU_EINVALID_AGG, "date_histogram requires `fixed_interval`");
          a.interval = parse_duration_ms(fi->s, false);
          if (const Json* off = spec.get("offset")) a.offset = off->is_str() ? parse_duration_ms(off->s, true) : off->as_f64();
        } else {
          a.interval = num_or(spec, "interval", 0);
          a.offset = num_or(spec, "offset", 0);
        }
        if (!(a.interval > 0)) fail(QWGPU_EINVALID_AGG, "histogram interval must be larger than 0");
        a.min_doc_count = (uint64_t)num_or(spec, "min_doc_count", 0);
        a.keyed = spec.bool_or("keyed", false);
        if (const Json* b = spec.get("hard_bounds")) { a.has_hard_bounds = true; a.hard_min = num_or(*b, "min", -INFINITY); a.hard_max = num_or(*b, "max", INFINITY); }
        if (const Json* b = spec.get("extended_bounds")) {
          a.has_extended_bounds = true; a.ext_min = num_or(*b, "min", INFINITY); a.ext_max = num_or(*b, "max", -INFINITY);
          if (a.min_doc_count > 0) fail(QWGPU_EINVALID_AGG, "Cannot set min_doc_count and extended_bounds at the same time");
        }
      } else if (t == "range") {
        a.kind = AggReq::Range;
        const Json* rs = spec.get("ranges");
        if (!rs || !rs->is_arr()) fail(QWGPU_EINVALID_AGG, "range aggregation requires `ranges`");
        for (auto& r : rs->arr) {
          AggReq::R x;
          if (const Json* f = r.get("from")) if (f->is_num()) { x.has_from = true; x.from = f->as_f64(); }
          if (const Json* f = r.get("to")) if (f->is_num()) { x.has_to = true; x.to = f->as_f64(); }
          x.key = r.str_or("key", "");
          a.ranges.push_back(x);
        }
        a.keyed = spec.bool_or("keyed", false);
      } else if (t == "stats" || t == "avg" || t == "sum" || t == "min" || t == "max" || t == "value_count" || t == "count") {
        a.kind = t == "stats" ? AggReq::Stats : t == "avg" ? AggReq::Avg : t == "sum" ? AggReq::Sum
               : t == "min" ? AggReq::Min : t == "max" ? AggReq::Max : AggReq::Count;
        parse_metric_missing(spec, a, t.c_str());
      } else if (t == "percentiles") parse_percentiles(spec, a);
      else if (t == "cardinality" || t == "extended_stats" || t == "top_hits" || t == "filter")
        fail(QWGPU_EUNSUPPORTED, "`%s` aggregations are not implemented on the GPU path yet", t.c_str());
      else fail(QWGPU_EINVALID_AGG, "unknown aggregation type `%s`", t.c_str());
    }
    if (!found) fail(QWGPU_EINVALID_AGG, "aggregation `%s` has no type", a.name.c_str());
    if (a.is_metric() && !a.children.empty()) fail(QWGPU_EINVALID_AGG, "metric aggregation `%s` cannot have sub-aggregations", a.name.c_str());
    out.push_back(std::move(a));
  }
}

// QuickwitAggregations is a serde untagged enum (collector.rs:600-640): the FindTraceIdsCollector shape is tried
// first — an object with `num_traces` (usize), `trace_id_field_name` and `span_timestamp_field_name` (strings),
// other keys ignored — and anything else is read as a tantivy aggregation map
static bool parse_trace_ids(const Json& j, AggReq& a) {
  const Json *n = j.get("num_traces"), *t = j.get("trace_id_field_name"), *s = j.get("span_timestamp_field_name");
  if (!n || !t || !s || !t->is_str() || !s->is_str()) return false;
  if (n->type == Json::U64) a.num_traces = n->u;
  else if (n->type == Json::I64 && n->i >= 0) a.num_traces = (uint64_t)n->i;
  else return false;
  a.kind = AggReq::TraceIds;
  a.field = t->s;
  a.ts_field = s->s;
  a.size = (uint32_t)std::min<uint64_t>(a.num_traces, 0xFFFFFFFFu);
  return true;
}

std::vector<AggReq> parse_agg_request(const std::string& json) {
  std::vector<AggReq> out;
  const Json j = parse_json(json, QWGPU_EINVALID_AGG);
  AggReq tr;
  if (parse_trace_ids(j, tr)) { out.push_back(std::move(tr)); return out; }
  parse_agg_map(j, out, 0);
  return out;
}

// ---- lowering ------------------------------------------------------------------------------------------
static uint64_t f64_bound_to_mapped(uint32_t type, double v) {  // smallest mapped value whose f64 is >= v
  switch (type) {
    case QW_COL_F64: return f64_to_u64(v);
    case QW_COL_U64: case QW_COL_BOOL: return v <= 0 ? 0 : (v >= 18446744073709551615.0 ? ~0ull : (uint64_t)std::ceil(v));
    default: {
      double c = std::ceil(v);
      int64_t i = c <= -9223372036854775808.0 ? INT64_MIN : (c >= 9223372036854775807.0 ? INT64_MAX : (int64_t)c);
      return i64_to_u64(i);
    }
  }
}

// Exact order between two non-null integers / floats of any of the three numeric key types: -1, 0, 1
static int num_cmp(const CompKey& x, const CompKey& y) {
  auto ld = [](const CompKey& k) { return k.t == CompKey::I64 ? (long double)k.i : k.t == CompKey::U64 ? (long double)k.u : (long double)k.f; };
  if (x.t == CompKey::F64 || y.t == CompKey::F64) {
    const long double a = ld(x), b = ld(y);  // (64-bit mantissa: every i64 / u64 is exact)
    if (std::isnan(a) || std::isnan(b)) return std::isnan(a) - std::isnan(b);
    return a < b ? -1 : (a > b ? 1 : 0);
  }
  if (x.t == y.t) return x.t == CompKey::I64 ? (x.i < y.i ? -1 : x.i > y.i) : (x.u < y.u ? -1 : x.u > y.u);
  if (x.t == CompKey::I64) return x.i < 0 ? -1 : ((uint64_t)x.i < y.u ? -1 : (uint64_t)x.i > y.u);
  return y.i < 0 ? 1 : (x.u < (uint64_t)y.i ? -1 : x.u > (uint64_t)y.i);
}
// Ascending order of one key position: null first, then bool, string (bytes), number (by value); keys of
// different columns types only meet when one field has different types in different splits
static int key_cmp(const CompKey& x, const CompKey& y) {
  const int rx = x.numeric() ? 3 : (int)x.t, ry = y.numeric() ? 3 : (int)y.t;
  if (rx != ry) return rx < ry ? -1 : 1;
  switch (rx) {
    case CompKey::Null: return 0;
    case CompKey::Bool: return x.u < y.u ? -1 : x.u > y.u;
    case CompKey::Str: { const int c = x.s.compare(y.s); return c < 0 ? -1 : c > 0; }
    default: return num_cmp(x, y);
  }
}

// The key of histogram position `pos` of a composite source: the histogram aggregation's bucket key
// (pos * interval + offset, in request units); a date_histogram key is the i64 of its epoch milliseconds
static CompKey comp_hist_key(const QwAggNode& n, uint32_t col_type, bool date, int64_t pos) {
  const double unit = col_type == QW_COL_DATETIME ? 1e6 : 1.0;
  CompKey c;
  c.f = ((double)pos * n.interval + n.offset) / unit;
  if (date) { c.t = CompKey::I64; c.i = (int64_t)std::llround(c.f); }
  else c.t = CompKey::F64;
  return c;
}

// The key space bound of one composite source node for its `after` value on this split (QwAggNode doc in
// qwgpu_format.h): false when the split's column cannot hold a key of after's type (the host filters alone then).
static bool comp_after_bound(const QwAggNode& n, const QwImgColumn* col, const ImageView& img, const AggReq& s, const CompKey& k,
                             uint64_t& bound, uint32_t& flags) {
  const bool desc = s.order_desc;
  bound = 0;
  if (k.t == CompKey::Null) { flags |= QW_AGG_COMP_AFTER_NULL; return true; }
  const uint64_t nb = n.num_buckets - (n.has_missing ? 1u : 0u);
  if (!col || !col->num_vals || nb == 0) { flags |= QW_AGG_COMP_AFTER_ALL; return true; }  // only null keys here
  bool exact = false;
  if (n.kind == QW_AGG_HISTOGRAM) {
    const double unit = col->type == QW_COL_DATETIME ? 1e6 : 1.0;
    auto key = [&](int64_t p) { return comp_hist_key(n, col->type, s.kind == AggReq::DateHistogram, p); };
    const double pos = qw_hist_pos((k.t == CompKey::F64 ? k.f : k.t == CompKey::I64 ? (double)k.i : (double)k.u) * unit, n.offset, n.interval);
    if (!std::isfinite(pos) || std::fabs(pos) > 9e15) return false;
    // the position from the formula, corrected by a few steps for the rounding of key(); keys that stay equal over
    // more positions than that (an offset far larger than the interval) leave the filter to the host
    int64_t q = (int64_t)pos;
    int steps = 0;
    if (!desc) {  // smallest position whose key is >= after
      while (num_cmp(key(q), k) < 0 && steps++ < 4) q++;
      while (num_cmp(key(q - 1), k) >= 0 && steps++ < 8) q--;
      if (num_cmp(key(q), k) < 0 || num_cmp(key(q - 1), k) >= 0) return false;
    } else {      // largest position whose key is <= after
      while (num_cmp(key(q), k) > 0 && steps++ < 4) q--;
      while (num_cmp(key(q + 1), k) <= 0 && steps++ < 8) q++;
      if (num_cmp(key(q), k) > 0 || num_cmp(key(q + 1), k) <= 0) return false;
    }
    exact = num_cmp(key(q), k) == 0;
    const int64_t idx = q - n.base_pos;
    if (!desc) {
      if (idx < 0) { bound = 0; exact = false; }
      else if ((uint64_t)idx >= nb) { flags |= QW_AGG_COMP_AFTER_ALL; return true; }
      else bound = (uint64_t)idx;
    } else {
      if (idx < 0) { flags |= QW_AGG_COMP_AFTER_ALL; return true; }
      else if ((uint64_t)idx >= nb) { bound = nb - 1; exact = false; }
      else bound = (uint64_t)idx;
    }
    if (exact) flags |= QW_AGG_COMP_EXACT;
    return true;
  }
  // TERMS: the after value in the column's mapped space (desc: the largest mapped value <= after, else the smallest >=)
  uint64_t m = 0;
  if (col->type == QW_COL_STR) {
    if (k.t != CompKey::Str) return false;
    const uint32_t lb = img.dict_lower_bound(*col, (const uint8_t*)k.s.data(), (uint32_t)k.s.size(), &exact);
    if (!desc) { if (lb >= col->dict_num_terms) { flags |= QW_AGG_COMP_AFTER_ALL; return true; } m = lb; }
    else if (exact) m = lb;
    else { if (lb == 0) { flags |= QW_AGG_COMP_AFTER_ALL; return true; } m = lb - 1; }
  } else if (col->type == QW_COL_BOOL) {
    if (k.t != CompKey::Bool) return false;
    m = k.u;
    exact = true;
  } else {
    if (!k.numeric()) return false;
    // the key type of the column's values, and the mapped value of the nearest one on the side that is kept
    const bool is_f = col->type == QW_COL_F64, is_i = col->type == QW_COL_I64 || col->type == QW_COL_DATETIME;
    CompKey lo_t, hi_t;  // the column type's range
    if (is_f) {
      if (k.t == CompKey::F64 && std::isnan(k.f)) return false;
      const double v = k.t == CompKey::F64 ? k.f : (k.t == CompKey::I64 ? (double)k.i : (double)k.u);
      CompKey c; c.t = CompKey::F64; c.f = v;
      const int cmp = num_cmp(c, k);  // the double nearest `after`, and where it lies
      double w = v;
      if (!desc && cmp < 0) w = std::nextafter(v, INFINITY);
      if (desc && cmp > 0) w = std::nextafter(v, -INFINITY);
      m = f64_to_u64(w == 0.0 ? 0.0 : w);
      exact = cmp == 0;
    } else {
      // integers: clamp `after` into the type's range, rounding towards the kept side
      long double v = k.t == CompKey::I64 ? (long double)k.i : k.t == CompKey::U64 ? (long double)k.u : (long double)k.f;
      const long double lo = is_i ? -9223372036854775808.0L : 0.0L, hi = is_i ? 9223372036854775807.0L : 18446744073709551615.0L;
      long double r = desc ? std::floor(v) : std::ceil(v);
      exact = r == v && v >= lo && v <= hi;
      if (r < lo) { if (desc) { flags |= QW_AGG_COMP_AFTER_ALL; return true; } r = lo; }
      if (r > hi) { if (!desc) { flags |= QW_AGG_COMP_AFTER_ALL; return true; } r = hi; }
      m = is_i ? i64_to_u64((int64_t)r) : (uint64_t)r;
    }
  }
  // mapped -> bit-packed raw (raw = (mapped - min) / gcd), rounding towards the kept side
  if (!desc) {
    if (m > col->max_value) { flags |= QW_AGG_COMP_AFTER_ALL; return true; }
    if (m < col->min_value) { bound = 0; exact = false; }
    else {
      const uint64_t d = m - col->min_value;
      bound = d / col->gcd + (d % col->gcd ? 1 : 0);
      exact = exact && d % col->gcd == 0;
    }
  } else {
    if (m < col->min_value) { flags |= QW_AGG_COMP_AFTER_ALL; return true; }
    if (m > col->max_value) { bound = (col->max_value - col->min_value) / col->gcd; exact = false; }
    else {
      const uint64_t d = m - col->min_value;
      bound = d / col->gcd;
      exact = exact && d % col->gcd == 0;
    }
  }
  if (exact) flags |= QW_AGG_COMP_EXACT;
  return true;
}

static QwAggNode lower_one(const AggReq& a, const ImageView& img, AggBinding& b, uint32_t comp_level = 0);
// source `level` of composite `a`: the source's own node, with the composite descriptor
static QwAggNode lower_comp_source(const AggReq& a, const ImageView& img, AggBinding& b, uint32_t level) {
  const AggReq& s = a.sources[level];
  QwAggNode n = lower_one(s, img, b);
  if (b.column >= 0 && img.columns[b.column].type == QW_COL_IP)
    fail(QWGPU_EUNSUPPORTED, "composite sources on ip field `%s` are not supported on the GPU path", s.field.c_str());
  b.req = &a;
  b.comp_level = level;
  if (s.has_missing && n.kind == QW_AGG_HISTOGRAM) n.num_buckets++;  // the missing bucket, last (as terms)
  n.has_missing = s.has_missing;
  uint32_t flags = QW_AGG_COMP_LEVEL | (level + 1 == a.sources.size() ? (uint32_t)QW_AGG_COMP_LAST : 0u) |
                   (s.order_desc ? (uint32_t)QW_AGG_COMP_DESC : 0u) | (s.has_missing ? (uint32_t)QW_AGG_COMP_MISSING : 0u);
  if (a.has_after && b.column >= 0 && a.after[level].t != CompKey::Null) {
    // a terms source's `after` value must have its column's key type (histogram sources were checked at parse time)
    const uint32_t ct = img.columns[b.column].type;
    const CompKey& k = a.after[level];
    if ((ct == QW_COL_STR && k.t != CompKey::Str) || (ct == QW_COL_BOOL && k.t != CompKey::Bool) ||
        (ct != QW_COL_STR && ct != QW_COL_BOOL && !k.numeric()))
      fail(QWGPU_EINVALID_AGG, "composite `after` value of source `%s` does not match the type of field `%s`", s.name.c_str(), s.field.c_str());
  }
  uint64_t bound = 0;
  if (a.has_after && comp_after_bound(n, b.column >= 0 ? &img.columns[b.column] : nullptr, img, s, a.after[level], bound, flags))
    flags |= QW_AGG_COMP_HAS_AFTER;
  n.reserved = flags;
  n.range_from[0] = bound;
  n.range_to[0] = a.size;
  return n;
}

static QwAggNode lower_one(const AggReq& a, const ImageView& img, AggBinding& b, uint32_t comp_level) {
  if (a.kind == AggReq::Composite) return lower_comp_source(a, img, b, comp_level);
  QwAggNode n;
  memset(&n, 0, sizeof n);
  n.parent = 0xFFFFFFFFu;
  n.column = 0xFFFFFFFFu;
  b.req = &a;
  int c = img.find_column(a.field);
  b.column = c;
  const QwImgColumn* col = c >= 0 ? &img.columns[c] : nullptr;
  if (col) { n.column = (uint32_t)c; b.col_type = col->type; }
  if (a.kind == AggReq::TraceIds) {
    // the engine fails the split when the trace-id column is absent or not a bytes column (for_segment's error)
    // and when the timestamp column exists but is not a date column; an absent timestamp column reads 0
    if (a.num_traces > QW_MAX_TOPK) fail(QWGPU_EUNSUPPORTED, "find_trace_ids with num_traces = %llu exceeds the GPU limit %d", (unsigned long long)a.num_traces, QW_MAX_TOPK);
    n.kind = QW_AGG_TRACE_IDS;
    n.num_buckets = (uint32_t)a.num_traces;
    const int tc = img.find_column(a.ts_field);
    n.reserved = tc >= 0 ? (uint32_t)tc : 0xFFFFFFFFu;
    return n;
  }
  if (col && col->type == QW_COL_BYTES) fail(QWGPU_EUNSUPPORTED, "aggregations on bytes field `%s` are not supported on the GPU path", a.field.c_str());
  if (col && col->type == QW_COL_IP && a.kind != AggReq::Terms)
    fail(QWGPU_EUNSUPPORTED, "only terms aggregations on ip field `%s` are supported on the GPU path", a.field.c_str());
  switch (a.kind) {
    case AggReq::Terms: {
      n.kind = QW_AGG_TERMS;
      // dense space beyond QW_AGG_DENSE_MAX_TERMS slots: the plan takes the hashed layout, where the bucket key is
      // the raw value itself and num_buckets only has to exceed that limit (saturated at 0xFFFFFFFF)
      uint64_t span = col ? (col->max_value - col->min_value) / col->gcd : 0;
      uint64_t nb = col && col->num_vals ? std::min<uint64_t>(span, 0xFFFFFFFEull) + 1 : 0;
      n.num_buckets = (uint32_t)std::min<uint64_t>(nb + (a.has_missing ? 1 : 0), 0xFFFFFFFFull);
      n.has_missing = a.has_missing;
      break;
    }
    case AggReq::Histogram: case AggReq::DateHistogram: {
      n.kind = QW_AGG_HISTOGRAM;
      if (col && col->type == QW_COL_STR) fail(QWGPU_EINVALID_AGG, "histogram on text field `%s`", a.field.c_str());
      if (a.kind == AggReq::DateHistogram && col && col->type != QW_COL_DATETIME)
        fail(QWGPU_EINVALID_AGG, "date_histogram requires a datetime field, `%s` is not", a.field.c_str());
      // DateTime columns hold nanoseconds: request values are milliseconds (aggregation.md:150-160)
      double scale = (col && col->type == QW_COL_DATETIME) ? 1e6 : 1.0;
      n.interval = a.interval * scale;
      n.offset = a.offset * scale;
      if (a.has_hard_bounds) { n.has_bounds = 1; n.bound_min = a.hard_min * scale; n.bound_max = a.hard_max * scale; }
      if (col && col->num_vals) {
        double lo = qw_mapped_to_f64(col->type, col->min_value), hi = qw_mapped_to_f64(col->type, col->max_value);
        if (n.has_bounds) { lo = std::max(lo, n.bound_min); hi = std::min(hi, n.bound_max); }
        if (lo <= hi) {
          double p0 = qw_hist_pos(lo, n.offset, n.interval), p1 = qw_hist_pos(hi, n.offset, n.interval);
          if (p1 - p0 + 1 > 65000.0 * 16) fail(QWGPU_EINVALID_AGG, "histogram would create too many buckets (%g)", p1 - p0 + 1);
          n.base_pos = (int64_t)p0;
          n.num_buckets = (uint32_t)(p1 - p0 + 1);
        }
      }
      break;
    }
    case AggReq::Range: {
      n.kind = QW_AGG_RANGE;
      if (a.ranges.size() > QW_MAX_AGG_RANGES) fail(QWGPU_EUNSUPPORTED, "more than %d ranges", QW_MAX_AGG_RANGES);
      n.num_ranges = n.num_buckets = (uint32_t)a.ranges.size();
      uint32_t t = col ? col->type : (uint32_t)QW_COL_F64;
      for (size_t i = 0; i < a.ranges.size(); i++) {
        n.range_from[i] = a.ranges[i].has_from ? f64_bound_to_mapped(t, a.ranges[i].from) : 0;
        n.range_to[i] = a.ranges[i].has_to ? f64_bound_to_mapped(t, a.ranges[i].to) : ~0ull;
      }
      break;
    }
    case AggReq::Percentiles: {
      // the bins of the split's boundary table for the column (the engine builds the table itself and checks the
      // count), one more for the `missing` entry
      n.kind = QW_AGG_PERCENTILES;
      if (col && col->type == QW_COL_STR) fail(QWGPU_EINVALID_AGG, "percentiles on text field `%s`", a.field.c_str());
      dds::Table t;
      if (col && !dds::column_table(*col, false, &t))
        fail(QWGPU_EUNSUPPORTED, "percentiles over field `%s`, which holds NaN or infinite values, are not implemented on the GPU path", a.field.c_str());
      n.num_buckets = (uint32_t)t.num_bins + (a.has_missing ? 1u : 0u);
      break;
    }
    default: n.kind = QW_AGG_STATS; n.num_buckets = 1; break;
  }
  if (n.kind == QW_AGG_STATS || n.kind == QW_AGG_PERCENTILES) {
    // the device only counts the docs without a value; the host folds the value in (metric_from_cell, build_percentiles_e)
    n.has_missing = a.has_missing;
    if (a.has_missing) { const double m = a.missing.as_f64(); memcpy(&n.missing_value, &m, 8); }
  }
  return n;
}

// A terms node over an `ip` field keys its buckets by address (IKey::Ip), whether or not this split holds the field's
// column: the field is `ip` when its column or its indexed field says so, or else the doc mapping.
static bool ip_binding(const AggReq& a, const ImageView& img, const AggBinding& b, const DocMapperInfo* dm) {
  if (b.column >= 0) return b.col_type == QW_COL_IP;
  const int f = img.find_field(a.field);
  if (f >= 0) return img.fields[f].tokenizer == QW_TOK_IP;
  if (dm) for (auto& fd : dm->fields) if (fd.name == a.field) return fd.type == "ip";
  return false;
}

std::vector<QwAggNode> lower_aggs(const std::vector<AggReq>& reqs, const ImageView& img, std::vector<AggBinding>& bindings,
                                  const DocMapperInfo* dm) {
  std::vector<QwAggNode> out;
  bindings.clear();
  struct Pending { const AggReq* a; uint32_t idx, level; };
  std::vector<Pending> queue;
  for (auto& a : reqs) {
    AggBinding b;
    out.push_back(lower_one(a, img, b));
    bindings.push_back(b);
    queue.push_back({&a, (uint32_t)out.size() - 1, 0});
  }
  for (size_t qi = 0; qi < queue.size(); qi++) {
    Pending p = queue[qi];
    if (p.a->kind == AggReq::Composite && p.level + 1 < p.a->sources.size()) {
      // a composite's sources form a chain: the next source is the only child
      out[p.idx].first_child = (uint32_t)out.size();
      out[p.idx].num_children = 1;
      AggBinding b;
      QwAggNode n = lower_one(*p.a, img, b, p.level + 1);
      n.parent = p.idx;
      out.push_back(n);
      bindings.push_back(b);
      queue.push_back({p.a, (uint32_t)out.size() - 1, p.level + 1});
      continue;
    }
    if (p.a->children.empty()) continue;
    out[p.idx].first_child = (uint32_t)out.size();
    out[p.idx].num_children = (uint32_t)p.a->children.size();
    for (auto& c : p.a->children) {
      AggBinding b;
      QwAggNode n = lower_one(c, img, b);
      n.parent = p.idx;
      out.push_back(n);
      bindings.push_back(b);
      queue.push_back({&c, (uint32_t)out.size() - 1, 0});
    }
  }
  // the walk filters a composite only when the split places `after` in the key space of every source; otherwise the
  // host alone filters and cuts it (AFTER_HOST)
  for (size_t i = 0; i < out.size(); i++) {
    const AggReq* r = bindings[i].req;
    if (r->kind != AggReq::Composite || bindings[i].comp_level != 0) continue;
    bool all = true;
    for (size_t j = i; j < out.size(); j++) if (bindings[j].req == r && !(out[j].reserved & QW_AGG_COMP_HAS_AFTER)) all = false;
    if (r->has_after && !all)
      for (size_t j = i; j < out.size(); j++)
        if (bindings[j].req == r) out[j].reserved = (out[j].reserved & ~(uint32_t)QW_AGG_COMP_HAS_AFTER) | QW_AGG_COMP_AFTER_HOST;
  }
  for (AggBinding& b : bindings) {
    const AggReq& a = b.req->kind == AggReq::Composite ? b.req->sources[b.comp_level] : *b.req;
    if (b.req->kind == AggReq::TraceIds || !ip_binding(a, img, b, dm)) continue;
    if (b.req->kind == AggReq::Composite) fail(QWGPU_EUNSUPPORTED, "composite sources on ip field `%s` are not supported on the GPU path", a.field.c_str());
    if (a.kind != AggReq::Terms) fail(QWGPU_EUNSUPPORTED, "only terms aggregations on ip field `%s` are supported on the GPU path", a.field.c_str());
    uint8_t addr[16];
    if (a.has_missing && !(a.missing.type == Json::Str && parse_ip_addr(a.missing.s, addr)))
      fail(QWGPU_EINVALID_AGG, "terms `missing` on ip field `%s` must be an IP address", a.field.c_str());
    b.ip = true;
  }
  return out;
}

// ---- intermediate model --------------------------------------------------------------------------------
struct IKey {
  // Ip: the 16 big-endian bytes of an IPv6 address in `s`; keys of one kind order by address
  enum K : uint8_t { Str = 0, F64 = 1, I64 = 2, U64 = 3, Ip = 4 } kind = Str;
  std::string s;
  double f = 0;
  int64_t i = 0;
  uint64_t u = 0;
  bool numeric() const { return kind == F64 || kind == I64 || kind == U64; }
  bool operator<(const IKey& o) const {
    if (kind != o.kind) {
      if (numeric() && o.numeric()) return num() < o.num();
      return kind < o.kind;
    }
    switch (kind) { case Str: case Ip: return s < o.s; case F64: return f < o.f; case I64: return i < o.i; default: return u < o.u; }
  }
  bool operator==(const IKey& o) const { return !(*this < o) && !(o < *this); }
  double num() const { return kind == F64 ? f : (kind == I64 ? (double)i : (double)u); }
};
struct IAgg;
struct IBucket {
  IKey key;        // terms
  double hkey = 0;  // histogram (column units) / range index
  std::vector<CompKey> ckey;  // composite: one key per source
  uint64_t count = 0;
  std::vector<IAgg> subs;
};
struct IAgg {
  uint8_t kind = 0;  // AggReq::Kind
  std::vector<IBucket> buckets;
  uint64_t sum_other = 0, error_bound = 0;
  uint8_t is_date = 0;
  // metric
  uint64_t m_count = 0;
  double m_sum = 0, m_min = INFINITY, m_max = -INFINITY;
  dds::Sketch sk;  // percentiles
  // key -> position in `buckets`, built on the first merge into this node and kept up to date, so that
  // folding n responses costs O(total buckets · log) instead of re-indexing the accumulator n times
  struct Index {
    std::map<IKey, size_t> terms;
    std::map<double, size_t> hist;
  };
  std::shared_ptr<Index> index;  // allocated on the first merge into this node (accumulators only)
};

struct BW {
  std::string out;
  void varint(uint64_t v) { while (v >= 0x80) { out += (char)(v | 0x80); v >>= 7; } out += (char)v; }
  void f64(double d) { out.append((const char*)&d, 8); }
  void str(const std::string& s) { varint(s.size()); out += s; }
};
struct BR {
  const uint8_t *p, *e;
  uint64_t varint() {
    uint64_t v = 0; int sh = 0;
    while (p < e) { uint8_t c = *p++; v |= (uint64_t)(c & 0x7F) << sh; if (!(c & 0x80)) return v; sh += 7; }
    fail(QWGPU_EINTERNAL, "failed to merge intermediate aggregation results: truncated buffer");
  }
  double f64() { if (e - p < 8) fail(QWGPU_EINTERNAL, "failed to merge intermediate aggregation results: truncated buffer"); double d; memcpy(&d, p, 8); p += 8; return d; }
  std::string str() { uint64_t n = varint(); if ((uint64_t)(e - p) < n) fail(QWGPU_EINTERNAL, "failed to merge intermediate aggregation results: truncated buffer"); std::string s((const char*)p, n); p += n; return s; }
};

static void ser_aggs(BW& w, const std::vector<IAgg>& v);
static void ser_agg(BW& w, const IAgg& a) {
  w.varint(a.kind);
  if (a.kind == AggReq::Composite) {
    // per bucket: the key tuple (type, value per source), doc_count, sub-aggregations
    w.varint(a.buckets.size());
    for (auto& b : a.buckets) {
      w.varint(b.ckey.size());
      for (const CompKey& k : b.ckey) {
        w.varint(k.t);
        switch (k.t) {
          case CompKey::Null: break;
          case CompKey::Str: w.str(k.s); break;
          case CompKey::I64: w.varint((uint64_t)k.i); break;
          case CompKey::F64: w.f64(k.f); break;
          default: w.varint(k.u);
        }
      }
      w.varint(b.count);
      ser_aggs(w, b.subs);
    }
    return;
  }
  if (a.kind == AggReq::Percentiles) {
    // min, max, then (zigzag bin ordinal, count) per non-empty bin in value order; the count is their sum
    w.f64(a.sk.min);
    w.f64(a.sk.max);
    w.varint(a.sk.bins.size());
    for (const auto& kv : a.sk.bins) { w.varint(((uint64_t)kv.first << 1) ^ (uint64_t)(kv.first >> 63)); w.varint(kv.second); }
    return;
  }
  if (a.kind >= AggReq::Stats) { w.varint(a.m_count); w.f64(a.m_sum); w.f64(a.m_min); w.f64(a.m_max); return; }
  w.varint(a.is_date);
  w.varint(a.sum_other);
  w.varint(a.error_bound);
  w.varint(a.buckets.size());
  for (auto& b : a.buckets) {
    if (a.kind == AggReq::Terms) {
      w.varint(b.key.kind);
      switch (b.key.kind) { case IKey::Str: case IKey::Ip: w.str(b.key.s); break; case IKey::F64: w.f64(b.key.f); break; case IKey::I64: w.varint((uint64_t)b.key.i); break; default: w.varint(b.key.u); }
    } else w.f64(b.hkey);
    w.varint(b.count);
    ser_aggs(w, b.subs);
  }
}
static void ser_aggs(BW& w, const std::vector<IAgg>& v) {
  w.varint(v.size());
  for (auto& a : v) ser_agg(w, a);
}
static std::vector<IAgg> de_aggs(BR& r);
static IAgg de_agg(BR& r) {
  IAgg a;
  a.kind = (uint8_t)r.varint();
  if (a.kind == AggReq::Composite) {
    const uint64_t n = r.varint();
    for (uint64_t i = 0; i < n; i++) {
      IBucket b;
      const uint64_t nk = r.varint();
      if (nk > (uint64_t)(r.e - r.p)) fail(QWGPU_EINTERNAL, "failed to merge intermediate aggregation results: truncated buffer");
      b.ckey.resize(nk);
      for (CompKey& k : b.ckey) {
        const uint64_t t = r.varint();
        if (t > CompKey::F64) fail(QWGPU_EINTERNAL, "failed to merge intermediate aggregation results: bad composite key");
        k.t = (CompKey::T)t;
        switch (k.t) {
          case CompKey::Null: break;
          case CompKey::Str: k.s = r.str(); break;
          case CompKey::I64: k.i = (int64_t)r.varint(); break;
          case CompKey::F64: k.f = r.f64(); break;
          default: k.u = r.varint();
        }
      }
      b.count = r.varint();
      b.subs = de_aggs(r);
      a.buckets.push_back(std::move(b));
    }
    return a;
  }
  if (a.kind == AggReq::Percentiles) {
    a.sk.min = r.f64();
    a.sk.max = r.f64();
    const uint64_t n = r.varint();
    if (n > (uint64_t)(r.e - r.p)) fail(QWGPU_EINTERNAL, "failed to merge intermediate aggregation results: truncated buffer");
    for (uint64_t i = 0; i < n; i++) {
      const uint64_t z = r.varint();
      const uint64_t c = r.varint();
      a.sk.bins[(int64_t)((z >> 1) ^ (~(z & 1) + 1))] += c;
      a.sk.count += c;
    }
    return a;
  }
  if (a.kind >= AggReq::Stats) { a.m_count = r.varint(); a.m_sum = r.f64(); a.m_min = r.f64(); a.m_max = r.f64(); return a; }
  a.is_date = (uint8_t)r.varint();
  a.sum_other = r.varint();
  a.error_bound = r.varint();
  uint64_t n = r.varint();
  for (uint64_t i = 0; i < n; i++) {
    IBucket b;
    if (a.kind == AggReq::Terms) {
      const uint64_t kk = r.varint();
      if (kk > IKey::Ip) fail(QWGPU_EINTERNAL, "failed to merge intermediate aggregation results: bad terms key");
      b.key.kind = (IKey::K)kk;
      switch (b.key.kind) { case IKey::Str: case IKey::Ip: b.key.s = r.str(); break; case IKey::F64: b.key.f = r.f64(); break; case IKey::I64: b.key.i = (int64_t)r.varint(); break; default: b.key.u = r.varint(); }
      if (b.key.kind == IKey::Ip && b.key.s.size() != 16) fail(QWGPU_EINTERNAL, "failed to merge intermediate aggregation results: bad ip key");
    } else b.hkey = r.f64();
    b.count = r.varint();
    b.subs = de_aggs(r);
    a.buckets.push_back(std::move(b));
  }
  return a;
}
static std::vector<IAgg> de_aggs(BR& r) {
  uint64_t n = r.varint();
  std::vector<IAgg> v;
  for (uint64_t i = 0; i < n; i++) v.push_back(de_agg(r));
  return v;
}
static const char kMagic[4] = {'Q', 'W', 'I', 'A'};
static std::string ser_top(const std::vector<IAgg>& v) {
  BW w;
  w.out.append(kMagic, 4);
  ser_aggs(w, v);
  return w.out;
}
static std::vector<IAgg> de_top(const std::string& s) {
  if (s.size() < 4 || memcmp(s.data(), kMagic, 4) != 0) fail(QWGPU_EINTERNAL, "failed to merge intermediate aggregation results: bad header");
  BR r{(const uint8_t*)s.data() + 4, (const uint8_t*)s.data() + s.size()};
  return de_aggs(r);
}

// ---- build a split's tree ------------------------------------------------------------------------------
static IKey term_key(const ImageView& img, const AggBinding& b, uint64_t raw, bool missing) {
  IKey k;
  if (missing && b.ip) {  // parsed when the plan was lowered
    uint8_t a[16];
    parse_ip_addr(b.req->missing.s, a);
    k.kind = IKey::Ip;
    k.s.assign((const char*)a, 16);
    return k;
  }
  if (missing) {
    const Json& m = b.req->missing;
    if (m.type == Json::Str) { k.kind = IKey::Str; k.s = m.s; }
    else if (m.type == Json::U64) { k.kind = IKey::U64; k.u = m.u; }
    else if (m.type == Json::I64) { k.kind = IKey::I64; k.i = m.i; }
    else { k.kind = IKey::F64; k.f = m.as_f64(); }
    return k;
  }
  const QwImgColumn& col = img.columns[b.column];
  uint64_t mapped = col.min_value + col.gcd * raw;
  switch (col.type) {
    case QW_COL_STR: { const uint8_t* p; uint32_t len; img.dict_term(col, (uint32_t)mapped, &p, &len); k.kind = IKey::Str; k.s.assign((const char*)p, len); break; }
    case QW_COL_IP: { const uint8_t* p; uint32_t len; img.dict_term(col, (uint32_t)mapped, &p, &len); k.kind = IKey::Ip; k.s.assign((const char*)p, len); break; }
    case QW_COL_F64: k.kind = IKey::F64; k.f = u64_to_f64(mapped); break;
    case QW_COL_I64: case QW_COL_DATETIME: k.kind = IKey::I64; k.i = u64_to_i64(mapped); break;
    default: k.kind = IKey::U64; k.u = mapped; break;
  }
  if (k.kind == IKey::U64 && k.u <= (uint64_t)INT64_MAX) { k.kind = IKey::I64; k.i = (int64_t)k.u; }
  return k;
}

static double metric_of(const IAgg& a, const std::string& prop) {
  if (a.kind < AggReq::Stats) return 0;
  std::string p = prop;
  if (p.empty()) p = a.kind == AggReq::Avg ? "avg" : a.kind == AggReq::Sum ? "sum" : a.kind == AggReq::Min ? "min" : a.kind == AggReq::Max ? "max" : a.kind == AggReq::Count ? "count" : "avg";
  if (p == "avg") return a.m_count ? a.m_sum / (double)a.m_count : 0;
  if (p == "sum") return a.m_sum;
  if (p == "min") return a.m_min;
  if (p == "max") return a.m_max;
  return (double)a.m_count;
}

// the requested order of term buckets (ties: key ascending, for determinism) as a permutation of their indices:
// std::sort makes the same comparisons on indices as on the buckets themselves, so the order is the same, and no
// (large) bucket moves
static std::vector<uint32_t> term_order(const AggReq& req, const std::vector<IBucket>& bs) {
  std::vector<uint32_t> perm(bs.size());
  for (size_t i = 0; i < perm.size(); i++) perm[i] = (uint32_t)i;
  auto sort_by = [&](auto less) {
    std::sort(perm.begin(), perm.end(), [&](uint32_t x, uint32_t y) { return less(bs[x], bs[y]); });
    return perm;
  };
  if (req.order_target == "_key")
    return sort_by([&](const IBucket& a, const IBucket& b) { return req.order_desc ? b.key < a.key : a.key < b.key; });
  if (req.order_target == "_count") {
    return sort_by([&](const IBucket& a, const IBucket& b) {
      if (a.count != b.count) return req.order_desc ? a.count > b.count : a.count < b.count;
      return a.key < b.key;
    });
  }
  std::string name = req.order_target, prop;
  size_t dot = name.find('.');
  if (dot != std::string::npos) { prop = name.substr(dot + 1); name = name.substr(0, dot); }
  int ci = -1;
  for (size_t i = 0; i < req.children.size(); i++) if (req.children[i].name == name) ci = (int)i;
  if (ci < 0) fail(QWGPU_EINVALID_AGG, "could not find aggregation with name `%s` in metric sub_aggregations", name.c_str());
  if (req.children[ci].kind == AggReq::Percentiles)
    fail(QWGPU_EUNSUPPORTED, "ordering terms by the percentiles aggregation `%s` is not implemented on the GPU path", name.c_str());
  return sort_by([&](const IBucket& a, const IBucket& b) {
    double x = metric_of(a.subs[ci], prop), y = metric_of(b.subs[ci], prop);
    if (x != y) return req.order_desc ? x > y : x < y;
    return a.key < b.key;
  });
}

// metric node ni from its cell (a cell with count 0 where no value reached it) and, with `missing`, the count of matched
// docs without a value under the same parent: each of those counts once as the `missing` value, an f64 in the space
// qw_mapped_to_f64 gives the column's values. On the exact route an integer `missing` that an i64 holds joins the
// 128-bit sum, rounded once; otherwise n * missing is added in f64 after the column's sum.
static IAgg metric_from_cell(const CompiledPlan& cp, const ImageView& img, const QwAggNode* nodes, uint32_t ni, const QwAggCell& cell,
                             uint64_t n_missing) {
  const AggBinding& b = cp.agg_bindings[ni];
  IAgg a;
  a.kind = (uint8_t)b.req->kind;
  a.m_count = cell.count + n_missing;
  const double m = n_missing ? b.req->missing.as_f64() : 0.0;
  const bool m_int = n_missing && m == std::trunc(m) && m >= -0x1p63 && m < 0x1p63;
  bool folded = false;
  if (cell.count && b.column >= 0) {
    uint32_t t = b.col_type;
    const QwImgColumn& col = img.columns[b.column];
    if (!qw_stats_sum_exact(img.columns, nodes, ni)) memcpy(&a.m_sum, &cell.sum_bits, 8);
    else {
      // exact: sum of the typed values = count * min + gcd * (sum of raw offsets); the mapped u64 of an
      // i64 / datetime is value + 2^63
      __int128 sum = (__int128)(unsigned __int128)col.min_value * (__int128)cell.count + (__int128)((unsigned __int128)col.gcd * cell.sum_bits);
      if (!(t == QW_COL_U64 || t == QW_COL_BOOL)) sum -= ((__int128)1 << 63) * (__int128)cell.count;
      // (|missing| <= 2^63 and n < 2^64 keep n * missing inside 128 bits)
      if (m_int) { sum += (__int128)(int64_t)m * (__int128)n_missing; folded = true; }
      a.m_sum = (double)sum;
    }
    a.m_min = qw_mapped_to_f64(t, cell.min_mapped);
    a.m_max = qw_mapped_to_f64(t, cell.max_mapped);
  }
  if (n_missing) {
    if (!folded) a.m_sum += (double)n_missing * m;
    if (m < a.m_min || !cell.count) a.m_min = m;
    if (m > a.m_max || !cell.count) a.m_max = m;
  }
  return a;
}

// per-split cut of a terms node to segment_size (cut_off_buckets): error bound = doc count of the first dropped
// bucket, sum_other = sum of dropped doc counts
static void cut_terms(const AggReq& req, IAgg& a) {
  if (req.kind == AggReq::Terms && req.order_target.find('.') == std::string::npos &&
      (req.order_target == "_count" || req.order_target == "_key")) {
    const std::vector<uint32_t> order = term_order(req, a.buckets);
    const size_t keep = std::min<size_t>(order.size(), req.segment_size);
    if (order.size() > keep && req.order_target == "_count" && req.order_desc) a.error_bound = a.buckets[order[keep]].count;
    std::vector<IBucket> kept;
    kept.reserve(keep);
    for (size_t i = 0; i < order.size(); i++) {
      if (i < keep) kept.push_back(std::move(a.buckets[order[i]]));
      else a.sum_other += a.buckets[order[i]].count;
    }
    a.buckets.swap(kept);
  }
}

// ---- composite: key order, the `after` filter and the cut to `size` (per split and after every merge) ---------
static int comp_cmp(const AggReq& req, const std::vector<CompKey>& x, const std::vector<CompKey>& y) {
  for (size_t i = 0; i < x.size() && i < y.size(); i++) {
    const int c = key_cmp(x[i], y[i]);
    if (c) return req.sources[i].order_desc ? -c : c;
  }
  return x.size() < y.size() ? -1 : x.size() > y.size();
}
struct CompKeyLess {  // source-order-free total order (merging by key tuple)
  bool operator()(const std::vector<CompKey>& x, const std::vector<CompKey>& y) const {
    for (size_t i = 0; i < x.size() && i < y.size(); i++) if (const int c = key_cmp(x[i], y[i])) return c < 0;
    return x.size() < y.size();
  }
};
static void comp_sort_cut(const AggReq& req, IAgg& a) {
  for (const IBucket& b : a.buckets)
    if (b.ckey.size() != req.sources.size()) fail(QWGPU_EINTERNAL, "intermediate aggregation result does not match the request");
  if (req.has_after)
    a.buckets.erase(std::remove_if(a.buckets.begin(), a.buckets.end(), [&](const IBucket& b) { return comp_cmp(req, b.ckey, req.after) <= 0; }),
                    a.buckets.end());
  std::sort(a.buckets.begin(), a.buckets.end(), [&](const IBucket& x, const IBucket& y) { return comp_cmp(req, x.ckey, y.ckey) < 0; });
  if (a.buckets.size() > req.size) a.buckets.resize(req.size);
}

// ---- build from entries (QwAggEntry) ------------------------------------------------------------------------
// A split's IAgg tree is built from entries whichever layout its result came in (dense cells become the entries of
// their nonzero cells): buckets in dense order (terms by raw key with `missing` last, histograms by position, every
// range in request order, empty ones included).
static const QwAggNode* plan_agg_nodes(const CompiledPlan& cp) {
  return (const QwAggNode*)(cp.bytes.data() + sizeof(QwPlanHeader) + (size_t)cp.header.num_nodes * sizeof(QwPlanNode));
}

struct EntryCtx {
  const CompiledPlan& cp;
  const ImageView& img;
  const QwAggNode* nodes;
  const QwAggEntry* entries;
  // entries grouped by (parent entry, node), each group in entry order: group g is members[start[g] .. start[g + 1]).
  // A top-level node's group is its node index; child node first_child + k of entry e's node has group first_group[e] + k.
  std::vector<size_t> first_group, start;
  std::vector<uint32_t> members;
};
static const uint32_t kNoEntry = 0xFFFFFFFEu;  // the parent of an empty range bucket: has no entries below it

static size_t entry_group(const EntryCtx& c, uint32_t ni, uint32_t parent) {
  return parent == QW_AGG_NO_PARENT ? ni : c.first_group[parent] + (ni - c.nodes[c.entries[parent].node].first_child);
}
struct EntryRange {
  const uint32_t *b, *e;
  const uint32_t* begin() const { return b; }
  const uint32_t* end() const { return e; }
  bool empty() const { return b == e; }
};
// the entries of node ni under parent entry `parent`
static EntryRange kids(const EntryCtx& c, uint32_t ni, uint32_t parent) {
  if (parent == kNoEntry) return {nullptr, nullptr};
  const size_t g = entry_group(c, ni, parent);
  return {c.members.data() + c.start[g], c.members.data() + c.start[g + 1]};
}
// groups the entries by a counting sort, linear in the entries; each parent must be an entry of its node's parent node
static void index_entries(EntryCtx& c, size_t nentries) {
  size_t groups = c.cp.header.num_aggs;
  c.first_group.resize(nentries);
  for (size_t e = 0; e < nentries; e++) {
    c.first_group[e] = groups;
    groups += c.nodes[c.entries[e].node].num_children;
  }
  // start[g] counts group g, then becomes its end, then (filled from the back) its begin
  c.start.assign(groups + 1, 0);
  for (size_t e = 0; e < nentries; e++) c.start[entry_group(c, c.entries[e].node, c.entries[e].parent)]++;
  for (size_t g = 1; g <= groups; g++) c.start[g] += c.start[g - 1];
  c.members.resize(nentries);
  for (size_t e = nentries; e-- > 0;) c.members[--c.start[entry_group(c, c.entries[e].node, c.entries[e].parent)]] = (uint32_t)e;
}

static IAgg build_node_e(const EntryCtx& c, uint32_t ni, uint32_t parent);

// the typed key of a composite source's entry: strings through the dictionary, numbers through the column mapping,
// histogram positions to the histogram key (date_histogram: epoch milliseconds)
static CompKey comp_entry_key(const EntryCtx& c, uint32_t ni, const QwAggEntry& x) {
  const QwAggNode& n = c.nodes[ni];
  const AggBinding& b = c.cp.agg_bindings[ni];
  CompKey k;
  if (x.flags & QW_AGG_ENTRY_MISSING) return k;
  const QwImgColumn& col = c.img.columns[b.column];
  if (n.kind == QW_AGG_HISTOGRAM) return comp_hist_key(n, col.type, b.req->sources[b.comp_level].kind == AggReq::DateHistogram, n.base_pos + (int64_t)x.key);
  const uint64_t mapped = col.min_value + col.gcd * x.key;
  switch (col.type) {
    case QW_COL_STR: { const uint8_t* p; uint32_t len; c.img.dict_term(col, (uint32_t)mapped, &p, &len); k.t = CompKey::Str; k.s.assign((const char*)p, len); break; }
    case QW_COL_F64: k.t = CompKey::F64; k.f = u64_to_f64(mapped); break;
    case QW_COL_I64: case QW_COL_DATETIME: k.t = CompKey::I64; k.i = u64_to_i64(mapped); break;
    case QW_COL_BOOL: k.t = CompKey::Bool; k.u = mapped; break;
    default: k.t = CompKey::U64; k.u = mapped; break;
  }
  return k;
}
// composite rooted at source node ni0: one bucket per leaf entry of the source chain, keyed by the chain's keys;
// then the `after` filter, the sort and the cut to `size`
static IAgg build_composite_e(const EntryCtx& c, uint32_t ni0, uint32_t parent0) {
  const AggReq& req = *c.cp.agg_bindings[ni0].req;
  IAgg a;
  a.kind = AggReq::Composite;
  std::vector<CompKey> path(req.sources.size());
  auto walk = [&](auto&& self, uint32_t ni, uint32_t parent, size_t level) -> void {
    const QwAggNode& n = c.nodes[ni];
    for (uint32_t e : kids(c, ni, parent)) {
      const QwAggEntry& x = c.entries[e];
      if (x.cell.count == 0) continue;
      path[level] = comp_entry_key(c, ni, x);
      if (level + 1 < path.size()) { self(self, n.first_child, e, level + 1); continue; }
      IBucket bk;
      bk.ckey = path;
      bk.count = x.cell.count;
      for (uint32_t k = 0; k < n.num_children; k++) bk.subs.push_back(build_node_e(c, n.first_child + k, e));
      a.buckets.push_back(std::move(bk));
    }
  };
  walk(walk, ni0, parent0, 0);
  comp_sort_cut(req, a);
  return a;
}

// a percentiles node's entries under one parent bucket as a sketch in value space: table indices become bin ordinals
// through the split's table for the column (tables differ per split, the ordinals do not); the `missing` entry counts
// the missing value
static IAgg build_percentiles_e(const EntryCtx& c, uint32_t ni, EntryRange es) {
  const AggBinding& b = c.cp.agg_bindings[ni];
  IAgg a;
  a.kind = AggReq::Percentiles;
  dds::Table t;
  const QwImgColumn* col = b.column >= 0 ? &c.img.columns[b.column] : nullptr;
  if (col) dds::column_table(*col, false, &t);
  for (uint32_t e : es) {
    const QwAggEntry& x = c.entries[e];
    if (x.flags & QW_AGG_ENTRY_MISSING) {
      const double m = b.req->missing.as_f64();
      a.sk.add(dds::bin_ord(m), x.cell.count, m, m);
    } else if (x.cell.count) {
      a.sk.add(t.ord_lo + (int64_t)x.key, x.cell.count, qw_mapped_to_f64(col->type, x.cell.min_mapped), qw_mapped_to_f64(col->type, x.cell.max_mapped));
    }
  }
  return a;
}

static IAgg build_node_e(const EntryCtx& c, uint32_t ni, uint32_t parent) {
  const QwAggNode& n = c.nodes[ni];
  const AggBinding& b = c.cp.agg_bindings[ni];
  const AggReq& req = *b.req;
  if (req.kind == AggReq::Composite) return build_composite_e(c, ni, parent);
  const EntryRange es = kids(c, ni, parent);
  if (req.kind == AggReq::Percentiles) return build_percentiles_e(c, ni, es);
  if (req.is_metric()) {
    // the node's cell and, with `missing`, its QW_AGG_ENTRY_MISSING entry: either may be absent
    QwAggCell cell = {0, 0, ~0ull, 0};
    uint64_t n_missing = 0;
    for (uint32_t e : es) {
      if (c.entries[e].flags & QW_AGG_ENTRY_MISSING) n_missing = c.entries[e].cell.count;
      else cell = c.entries[e].cell;
    }
    return metric_from_cell(c.cp, c.img, c.nodes, ni, cell, n_missing);
  }
  auto subs = [&](uint32_t e) {
    std::vector<IAgg> out;
    for (uint32_t k = 0; k < n.num_children; k++) out.push_back(build_node_e(c, n.first_child + k, e));
    return out;
  };
  IAgg a;
  a.kind = (uint8_t)req.kind;
  a.is_date = req.kind == AggReq::DateHistogram;
  if (req.kind == AggReq::Range) {
    for (uint32_t k = 0; k < n.num_ranges; k++) {
      uint32_t e = kNoEntry;
      for (uint32_t x : es) if (c.entries[x].key == k) e = x;
      IBucket bk;
      bk.count = e == kNoEntry ? 0 : c.entries[e].cell.count;
      bk.hkey = (double)k;
      bk.subs = subs(e);
      a.buckets.push_back(std::move(bk));
    }
    return a;
  }
  std::vector<uint32_t> order(es.begin(), es.end());
  auto before = [&](uint32_t x, uint32_t y) {
    const QwAggEntry &p = c.entries[x], &q = c.entries[y];
    const bool pm = p.flags & QW_AGG_ENTRY_MISSING, qm = q.flags & QW_AGG_ENTRY_MISSING;
    return pm != qm ? qm : p.key < q.key;
  };
  if (!std::is_sorted(order.begin(), order.end(), before)) std::sort(order.begin(), order.end(), before);
  a.buckets.reserve(order.size());
  for (uint32_t e : order) {
    const QwAggEntry& x = c.entries[e];
    if (x.cell.count == 0) continue;
    IBucket bk;
    bk.count = x.cell.count;
    if (req.kind == AggReq::Terms) bk.key = term_key(c.img, b, x.key, (x.flags & QW_AGG_ENTRY_MISSING) != 0);
    else bk.hkey = (double)(n.base_pos + (int64_t)x.key) * n.interval + n.offset;
    bk.subs = subs(e);
    a.buckets.push_back(std::move(bk));
  }
  cut_terms(req, a);
  return a;
}

static std::vector<IAgg> build_tree(const CompiledPlan& cp, const ImageView& img, const QwAggEntry* entries, size_t nentries) {
  EntryCtx c{cp, img, plan_agg_nodes(cp), entries, {}, {}, {}};
  index_entries(c, nentries);
  std::vector<IAgg> top;
  for (uint32_t i = 0; i < cp.header.num_aggs; i++) if (c.nodes[i].parent == 0xFFFFFFFFu) top.push_back(build_node_e(c, i, QW_AGG_NO_PARENT));
  return top;
}

// entries that come from outside the program: every one must name a bucket of its node's key space, once, under its parent
static std::vector<IAgg> build_top_entries(const CompiledPlan& cp, const ImageView& img, const QwAggEntry* entries, size_t nentries) {
  const QwPlanHeader& h = cp.header;
  const QwAggNode* nodes = plan_agg_nodes(cp);
  std::set<std::tuple<uint32_t, uint32_t, uint64_t, uint32_t>> seen;
  for (size_t e = 0; e < nentries; e++) {
    const QwAggEntry& x = entries[e];
    if (x.node >= h.num_aggs || (x.parent != QW_AGG_NO_PARENT && (x.parent >= nentries || entries[x.parent].node != nodes[x.node].parent)) ||
        (x.parent == QW_AGG_NO_PARENT && nodes[x.node].parent != 0xFFFFFFFFu))
      fail(QWGPU_EINVALID_ARG, "aggregation entry %zu does not match the plan's tree", e);
    const QwAggNode& n = nodes[x.node];
    const AggBinding& b = cp.agg_bindings[x.node];
    bool ok = x.flags == 0 || ((n.kind == QW_AGG_TERMS || n.kind == QW_AGG_HISTOGRAM || n.kind == QW_AGG_PERCENTILES || n.kind == QW_AGG_STATS) &&
                               x.flags == QW_AGG_ENTRY_MISSING);
    if (ok && (x.flags & QW_AGG_ENTRY_MISSING)) ok = n.has_missing && x.key == 0;
    else if (ok) {
      switch (n.kind) {
        case QW_AGG_STATS: ok = x.key == 0; break;
        case QW_AGG_HISTOGRAM: case QW_AGG_PERCENTILES: ok = x.key < (uint64_t)n.num_buckets - (n.has_missing ? 1u : 0u); break;
        case QW_AGG_RANGE: ok = x.key < n.num_ranges; break;
        case QW_AGG_TERMS: {
          ok = b.column >= 0 && img.columns[b.column].num_vals > 0 && img.columns[b.column].gcd &&
               x.key <= (img.columns[b.column].max_value - img.columns[b.column].min_value) / img.columns[b.column].gcd;
          const QwImgColumn& col = img.columns[b.column >= 0 ? b.column : 0];
          if (ok && (col.type == QW_COL_STR || col.type == QW_COL_IP)) ok = col.min_value + col.gcd * x.key < col.dict_num_terms;
          break;
        }
        default: ok = false;
      }
    }
    if (!ok) fail(QWGPU_EINVALID_ARG, "aggregation entry %zu: key %llu (flags %u) is not a bucket of node %u", e, (unsigned long long)x.key, x.flags, x.node);
    if (!seen.insert(std::make_tuple(x.parent, x.node, x.key, x.flags)).second)
      fail(QWGPU_EINVALID_ARG, "aggregation entry %zu repeats a bucket of node %u under the same parent", e, x.node);
  }
  return build_tree(cp, img, entries, nentries);
}

uint64_t agg_cell_layout(const QwAggNode* aggs, uint32_t n, std::vector<uint32_t>* bases) {
  uint64_t total = 0;
  if (bases) bases->resize(n);
  for (uint32_t i = 0; i < n; i++) {
    // a STATS node with `missing` has a second bank: the count of docs without a value per parent cell
    uint64_t cells = aggs[i].kind == QW_AGG_STATS ? (aggs[i].has_missing ? 2 : 1) : aggs[i].num_buckets;
    uint32_t p = aggs[i].parent;
    while (p != 0xFFFFFFFFu) { cells *= aggs[p].num_buckets; p = aggs[p].parent; }
    if (bases) (*bases)[i] = (uint32_t)total;
    total += cells;
    if (total > QW_AGG_DENSE_MAX_CELLS) fail(QWGPU_EINVALID_AGG, "aggregation bucket space too large (%llu cells)", (unsigned long long)total);
  }
  return total;
}

// Hashed layout: a cell exists per (node, parent cell, key) that some (doc, value path) reaches, so a node has at
// most min(its dense cells, the (doc, value path) tuples of its bucket chain) cells. A chain of single-valued
// columns gives at most one path per doc; a multi-valued level multiplies by that column's value count (Σ_d Π v_l(d)
// <= Π Σ_d v_l(d)), a `missing` bucket adds one value per doc, a range node every range. A STATS node with `missing`
// has its `missing` entry next to its cell under every parent.
static uint64_t sat_mul(uint64_t a, uint64_t b) {
  const uint64_t lim = 1ull << 62;
  return (b && a > lim / b) ? lim : std::min(a * b, lim);
}
uint64_t agg_hashed_bound(const QwAggNode* aggs, uint32_t n, const ImageView& img) {
  const uint64_t num_docs = img.hdr->num_docs;
  uint64_t total = 0;
  for (uint32_t i = 0; i < n; i++) {
    uint64_t dense = 1, reps = 1, multi = 1;
    bool any_multi = false;
    uint32_t depth = 0;
    for (uint32_t b = aggs[i].kind == QW_AGG_STATS ? aggs[i].parent : i; b != 0xFFFFFFFFu && depth <= n; b = aggs[b].parent, depth++) {
      const QwAggNode& g = aggs[b];
      dense = sat_mul(dense, g.num_buckets);
      if (g.kind == QW_AGG_RANGE) reps = sat_mul(reps, g.num_ranges);
      if (g.column < img.hdr->num_columns && img.columns[g.column].cardinality == QW_CARD_MULTI) {
        any_multi = true;
        multi = sat_mul(multi, img.columns[g.column].num_vals +
                                   ((g.kind == QW_AGG_TERMS || g.kind == QW_AGG_HISTOGRAM || g.kind == QW_AGG_PERCENTILES) && g.has_missing ? num_docs : 0));
      }
    }
    const uint64_t cells = std::min(dense, sat_mul(any_multi ? multi : num_docs, reps));
    total = std::min<uint64_t>(total + sat_mul(cells, aggs[i].kind == QW_AGG_STATS && aggs[i].has_missing ? 2 : 1), 1ull << 62);
  }
  return total;
}
uint32_t agg_hashed_slots(uint64_t cap) {
  uint64_t slots = 2;
  while (slots < 2 * cap) slots <<= 1;  // load factor <= 1/2: short probe sequences
  return (uint32_t)std::min<uint64_t>(slots, 1ull << 31);
}
uint64_t agg_hashed_table_bytes(uint64_t cap) {
  const uint64_t slots = agg_hashed_slots(cap);
  return slots * 4 + cap * (sizeof(DHKey) + sizeof(QwAggCell));
}
uint64_t agg_hashed_layout(const QwAggNode* aggs, uint32_t n, const ImageView& img, const char* split_id) {
  const uint64_t bound = std::max<uint64_t>(agg_hashed_bound(aggs, n, img), 1);
  const uint64_t bytes = bound >= (1ull << 30) ? ~0ull : agg_hashed_table_bytes(bound);
  if (bytes > QWGPU_HASHED_MAX_BYTES)
    fail(QWGPU_EUNSUPPORTED, "split `%s`: the aggregation may create up to %llu buckets, whose hashed table exceeds the GPU limit of %llu bytes per call",
         split_id, (unsigned long long)bound, (unsigned long long)QWGPU_HASHED_MAX_BYTES);
  return bound;
}

// The entries of a dense cell array (QwAggCell doc in qwgpu_format.h), parents before children: one per nonzero cell,
// keyed by its bucket index within the node (a node's `missing` bucket, its last, as QW_AGG_ENTRY_MISSING with key 0;
// a metric cell with key 0, and the count of its second bank as QW_AGG_ENTRY_MISSING with key 0). Zero cells give none:
// the builder puts back every empty range bucket and metric.
static std::vector<QwAggEntry> dense_entries(const CompiledPlan& cp, const QwAggCell* cells, size_t ncells) {
  const QwAggNode* nodes = plan_agg_nodes(cp);
  std::vector<uint32_t> bases;
  const uint64_t total = agg_cell_layout(nodes, cp.header.num_aggs, &bases);
  if (total != ncells) fail(QWGPU_EINTERNAL, "aggregation cell count mismatch (%llu vs %zu)", (unsigned long long)total, ncells);
  std::vector<QwAggEntry> out;
  out.reserve(std::min<size_t>(ncells, 4096));  // (larger results grow)
  auto walk = [&](auto&& self, uint32_t ni, uint32_t parent, uint64_t parent_cell) -> void {
    const AggReq::Kind kind = cp.agg_bindings[ni].req->kind;
    if (kind == AggReq::Composite || kind == AggReq::Percentiles) fail(QWGPU_EINVALID_ARG, "composite and percentiles aggregation results are given as entries");
    const QwAggNode& n = nodes[ni];
    const QwAggCell* base = cells + bases[ni];
    if (n.kind == QW_AGG_STATS) {
      if (base[parent_cell].count) out.push_back({ni, parent, 0, 0u, 0, base[parent_cell]});
      if (n.has_missing) {
        uint64_t parent_cells = 1;  // the first bank's size
        for (uint32_t p = n.parent; p != 0xFFFFFFFFu; p = nodes[p].parent) parent_cells *= nodes[p].num_buckets;
        const QwAggCell& m = base[parent_cells + parent_cell];
        if (m.count) out.push_back({ni, parent, 0, (uint32_t)QW_AGG_ENTRY_MISSING, 0, m});
      }
      return;
    }
    const uint32_t nb = n.num_buckets;
    for (uint32_t k = 0; k < nb; k++) {
      const uint64_t cell = parent_cell * nb + k;
      if (!base[cell].count) continue;
      const bool missing = n.has_missing && k == nb - 1;
      out.push_back({ni, parent, missing ? 0 : k, missing ? (uint32_t)QW_AGG_ENTRY_MISSING : 0u, 0, base[cell]});
      const uint32_t e = (uint32_t)out.size() - 1;
      for (uint32_t j = 0; j < n.num_children; j++) self(self, n.first_child + j, e, cell);
    }
  };
  for (uint32_t i = 0; i < cp.header.num_aggs; i++) if (nodes[i].parent == 0xFFFFFFFFu) walk(walk, i, QW_AGG_NO_PARENT, 0);
  return out;
}

static std::vector<IAgg> build_top_cells(const CompiledPlan& cp, const ImageView& img, const QwAggCell* cells, size_t ncells) {
  const std::vector<QwAggEntry> entries = dense_entries(cp, cells, ncells);
  return build_tree(cp, img, entries.data(), entries.size());
}

std::string build_intermediate_aggs_entries(const CompiledPlan& cp, const ImageView& img, const QwAggEntry* entries, size_t nentries) {
  if (is_trace_ids_request(cp.agg_request)) fail(QWGPU_EINVALID_ARG, "find_trace_ids results are not given as entries");
  return ser_top(build_top_entries(cp, img, entries, nentries));
}

// ---- find_trace_ids: spans, postcard bytes, merge_segment_fruits -----------------------------------------------
bool span_less(const TraceSpan& a, const TraceSpan& b) {
  if (a.ts != b.ts) return a.ts > b.ts;
  return memcmp(a.id, b.id, 16) < 0;
}

static void put_varint(std::string& o, uint64_t v) {
  while (v >= 0x80) { o.push_back((char)(uint8_t)(v | 0x80)); v >>= 7; }
  o.push_back((char)(uint8_t)v);
}
static uint64_t get_varint(const std::string& s, size_t& p) {
  uint64_t v = 0;
  for (int sh = 0; sh < 70; sh += 7) {
    if (p >= s.size()) fail(QWGPU_EINTERNAL, "failed to merge intermediate aggregation results: Postcard error: truncated varint");
    const uint8_t b = (uint8_t)s[p++];
    if (sh == 63 && b > 1) fail(QWGPU_EINTERNAL, "failed to merge intermediate aggregation results: Postcard error: varint overflow");
    v |= (uint64_t)(b & 0x7F) << sh;
    if (!(b & 0x80)) return v;
  }
  fail(QWGPU_EINTERNAL, "failed to merge intermediate aggregation results: Postcard error: varint too long");
}

std::string encode_spans(const std::vector<TraceSpan>& v) {
  std::string o;
  o.reserve(5 + v.size() * 26);
  put_varint(o, v.size());
  for (const TraceSpan& sp : v) {
    o.append((const char*)sp.id, 16);
    put_varint(o, ((uint64_t)sp.ts << 1) ^ (uint64_t)(sp.ts >> 63));  // zigzag
  }
  return o;
}

std::vector<TraceSpan> decode_spans(const std::string& s) {
  size_t p = 0;
  const uint64_t n = get_varint(s, p);
  if (n > s.size()) fail(QWGPU_EINTERNAL, "failed to merge intermediate aggregation results: Postcard error: bad length");
  std::vector<TraceSpan> v((size_t)n);
  for (TraceSpan& sp : v) {
    if (s.size() - p < 16) fail(QWGPU_EINTERNAL, "failed to merge intermediate aggregation results: Postcard error: truncated span");
    memcpy(sp.id, s.data() + p, 16);
    p += 16;
    const uint64_t z = get_varint(s, p);
    sp.ts = (int64_t)((z >> 1) ^ (~(z & 1) + 1));
  }
  if (p != s.size()) fail(QWGPU_EINTERNAL, "failed to merge intermediate aggregation results: Postcard error: trailing bytes");
  return v;
}

std::vector<TraceSpan> merge_span_fruits(std::vector<std::vector<TraceSpan>> fruits, uint64_t num_traces) {
  for (auto& f : fruits) std::sort(f.begin(), f.end(), span_less);
  // k-merge: equal spans (same timestamp and id) are interchangeable, so a stable heap order is not needed
  struct Head { size_t f, i; };
  auto worse = [&](const Head& a, const Head& b) { return span_less(fruits[b.f][b.i], fruits[a.f][a.i]); };
  std::vector<Head> heap;
  for (size_t f = 0; f < fruits.size(); f++) if (!fruits[f].empty()) heap.push_back({f, 0});
  std::make_heap(heap.begin(), heap.end(), worse);
  std::vector<TraceSpan> out;
  std::vector<std::string> seen;
  while (!heap.empty() && out.size() < num_traces) {
    std::pop_heap(heap.begin(), heap.end(), worse);
    Head h = heap.back();
    const TraceSpan& sp = fruits[h.f][h.i];
    std::string id((const char*)sp.id, 16);
    auto it = std::lower_bound(seen.begin(), seen.end(), id);
    if (it == seen.end() || *it != id) { seen.insert(it, id); out.push_back(sp); }
    if (++h.i < fruits[h.f].size()) { heap.back() = h; std::push_heap(heap.begin(), heap.end(), worse); }
    else heap.pop_back();
  }
  return out;
}

// the split's spans from the N cells of its QW_AGG_TRACE_IDS node (QwAggNode doc), sorted
static std::vector<TraceSpan> trace_spans_of(const CompiledPlan& cp, const ImageView& img, const QwAggCell* cells, size_t ncells) {
  const QwAggNode& n = plan_agg_nodes(cp)[0];
  if (ncells != n.num_buckets) fail(QWGPU_EINTERNAL, "aggregation cell count mismatch (%u vs %zu)", n.num_buckets, ncells);
  std::vector<TraceSpan> v;
  for (size_t j = 0; j < ncells; j++) {
    if (cells[j].count != 1) continue;
    if (n.column >= img.hdr->num_columns) fail(QWGPU_EINTERNAL, "find_trace_ids: trace id column missing");
    const QwImgColumn& col = img.columns[n.column];
    if (cells[j].sum_bits >= col.dict_num_terms) fail(QWGPU_EINTERNAL, "find_trace_ids: trace id ordinal out of range");
    const uint8_t* p;
    uint32_t len;
    img.dict_term(col, (uint32_t)cells[j].sum_bits, &p, &len);
    if (len != 16) fail(QWGPU_EINTERNAL, "find_trace_ids: trace id of %u bytes (16 expected)", len);
    TraceSpan sp;
    memcpy(sp.id, p, 16);
    sp.ts = u64_to_i64(cells[j].max_mapped);
    v.push_back(sp);
  }
  std::sort(v.begin(), v.end(), span_less);
  return v;
}

std::string build_intermediate_aggs(const CompiledPlan& cp, const ImageView& img, const QwAggCell* cells, size_t ncells) {
  // (a single split's spans go out sorted: the reference leaves them in select_nth_unstable order)
  if (is_trace_ids_request(cp.agg_request)) return encode_spans(trace_spans_of(cp, img, cells, ncells));
  return ser_top(build_top_cells(cp, img, cells, ncells));
}

// ---- merge ------------------------------------------------------------------------------------------------
static void merge_into(const AggReq& req, IAgg& acc, IAgg&& other);
static void merge_lists(const std::vector<AggReq>& reqs, std::vector<IAgg>& acc, std::vector<IAgg>&& other) {
  if (acc.empty()) { acc = std::move(other); return; }
  if (other.empty()) return;
  if (acc.size() != other.size() || acc.size() != reqs.size()) fail(QWGPU_EINTERNAL, "failed to merge intermediate aggregation results: shape mismatch");
  for (size_t i = 0; i < acc.size(); i++) merge_into(reqs[i], acc[i], std::move(other[i]));
}
static void merge_into(const AggReq& req, IAgg& acc, IAgg&& other) {
  if (acc.kind != other.kind) fail(QWGPU_EINTERNAL, "failed to merge intermediate aggregation results: kind mismatch");
  if (acc.kind == AggReq::Composite) {
    // union by key tuple, then the same filter / sort / cut as each split's. Exact: a bucket among the first `size`
    // of the merge has fewer than `size` buckets before it in any part, so no part's cut dropped it
    std::map<std::vector<CompKey>, size_t, CompKeyLess> index;
    for (size_t i = 0; i < acc.buckets.size(); i++) index.emplace(acc.buckets[i].ckey, i);
    for (auto& b : other.buckets) {
      auto it = index.find(b.ckey);
      if (it == index.end()) { index.emplace(b.ckey, acc.buckets.size()); acc.buckets.push_back(std::move(b)); }
      else { IBucket& t = acc.buckets[it->second]; t.count += b.count; merge_lists(req.children, t.subs, std::move(b.subs)); }
    }
    comp_sort_cut(req, acc);
    return;
  }
  if (acc.kind == AggReq::Percentiles) {  // bins add up; min and max of both
    acc.sk.merge(other.sk);
    return;
  }
  if (acc.kind >= AggReq::Stats) {
    acc.m_count += other.m_count;
    acc.m_sum += other.m_sum;
    acc.m_min = std::min(acc.m_min, other.m_min);
    acc.m_max = std::max(acc.m_max, other.m_max);
    return;
  }
  acc.sum_other += other.sum_other;
  acc.error_bound += other.error_bound;
  if (acc.kind == AggReq::Terms) {
    if (!acc.index) { acc.index = std::make_shared<IAgg::Index>(); for (size_t i = 0; i < acc.buckets.size(); i++) acc.index->terms[acc.buckets[i].key] = i; }
    auto& index = acc.index->terms;
    for (auto& b : other.buckets) {
      auto it = index.find(b.key);
      if (it == index.end()) { index[b.key] = acc.buckets.size(); acc.buckets.push_back(std::move(b)); }
      else { IBucket& t = acc.buckets[it->second]; t.count += b.count; merge_lists(req.children, t.subs, std::move(b.subs)); }
    }
  } else {
    if (!acc.index) { acc.index = std::make_shared<IAgg::Index>(); for (size_t i = 0; i < acc.buckets.size(); i++) acc.index->hist[acc.buckets[i].hkey] = i; }
    auto& index = acc.index->hist;
    for (auto& b : other.buckets) {
      auto it = index.find(b.hkey);
      if (it == index.end()) { index[b.hkey] = acc.buckets.size(); acc.buckets.push_back(std::move(b)); }
      else { IBucket& t = acc.buckets[it->second]; t.count += b.count; merge_lists(req.children, t.subs, std::move(b.subs)); }
    }
  }
}

// Leaf-level merge of the splits of one request straight from their cells or entries: what
// merge_intermediate_aggs(build_intermediate_aggs(split) ...) yields, without serialising every split's
// result only to parse it again.
std::string build_and_merge_intermediate_aggs(const std::vector<AggReq>& reqs, const std::vector<SplitAggCells>& splits) {
  if (is_trace_ids_request(reqs)) {
    std::vector<std::vector<TraceSpan>> fruits;
    for (const SplitAggCells& sp : splits) fruits.push_back(trace_spans_of(*sp.plan, *sp.img, sp.cells, sp.ncells));
    return encode_spans(merge_span_fruits(std::move(fruits), reqs[0].num_traces));
  }
  std::vector<IAgg> acc;
  for (const SplitAggCells& sp : splits) {
    std::vector<IAgg> top = sp.hashed ? build_top_entries(*sp.plan, *sp.img, sp.entries, sp.nentries) : build_top_cells(*sp.plan, *sp.img, sp.cells, sp.ncells);
    if (acc.empty() && !top.empty()) {
      // same normalisation as a serialise / parse round trip would apply: none needed — the first
      // split's tree becomes the accumulator
      acc = std::move(top);
      continue;
    }
    merge_lists(reqs, acc, std::move(top));
  }
  return ser_top(acc);
}

std::string merge_intermediate_aggs(const std::vector<AggReq>& reqs, const std::vector<std::string>& parts) {
  if (is_trace_ids_request(reqs)) {
    // merge_intermediate_aggregation_result / IncrementalCollector (collector.rs:640-704,871-886); staged merges of
    // the incremental collector give the same spans, so every part is merged at once
    std::vector<std::vector<TraceSpan>> fruits;
    for (auto& p : parts) fruits.push_back(decode_spans(p));
    return encode_spans(merge_span_fruits(std::move(fruits), reqs[0].num_traces));
  }
  std::vector<IAgg> acc;
  for (auto& p : parts) merge_lists(reqs, acc, de_top(p));
  return ser_top(acc);
}

// ---- finalize -----------------------------------------------------------------------------------------------
static void civil_from_days(int64_t z, int64_t* y, unsigned* m, unsigned* d) {
  z += 719468;
  const int64_t era = (z >= 0 ? z : z - 146096) / 146097;
  const unsigned doe = (unsigned)(z - era * 146097);
  const unsigned yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
  *y = (int64_t)yoe + era * 400;
  const unsigned doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
  const unsigned mp = (5 * doy + 2) / 153;
  *d = doy - (153 * mp + 2) / 5 + 1;
  *m = mp < 10 ? mp + 3 : mp - 9;
  *y += *m <= 2;
}
static std::string rfc3339_from_ms(double ms) {
  int64_t total_ms = (int64_t)std::floor(ms);
  int64_t secs = total_ms / 1000, rem = total_ms % 1000;
  if (rem < 0) { rem += 1000; secs -= 1; }
  int64_t days = secs / 86400, sod = secs % 86400;
  if (sod < 0) { sod += 86400; days -= 1; }
  int64_t y; unsigned m, d;
  civil_from_days(days, &y, &m, &d);
  char b[64];
  if (rem) snprintf(b, sizeof b, "%04lld-%02u-%02uT%02lld:%02lld:%02lld.%03lldZ", (long long)y, m, d, (long long)(sod / 3600), (long long)(sod % 3600 / 60), (long long)(sod % 60), (long long)rem);
  else snprintf(b, sizeof b, "%04lld-%02u-%02uT%02lld:%02lld:%02lldZ", (long long)y, m, d, (long long)(sod / 3600), (long long)(sod % 3600 / 60), (long long)(sod % 60));
  return b;
}

static void fin_aggs(const std::vector<AggReq>& reqs, const std::vector<IAgg>* aggs, std::string& out);

static void fin_key(const IKey& k, std::string& out) {
  switch (k.kind) {
    case IKey::Str: json_escape(k.s, out); break;
    case IKey::Ip: json_escape(format_ip_addr((const uint8_t*)k.s.data()), out); break;
    case IKey::F64: json_f64(k.f, out); break;
    case IKey::I64: out += std::to_string(k.i); break;
    default: out += std::to_string(k.u);
  }
}
// an f64 the way Rust's Display writes it: the shortest digits that read back the same value, never an exponent,
// no ".0" on whole numbers (100 -> "100", 0.1 -> "0.1", 1e21 -> "1000000000000000000000")
static std::string rust_display_f64(double v) {
  if (std::isnan(v)) return "NaN";
  if (std::isinf(v)) return v > 0 ? "inf" : "-inf";
  char buf[64];
  for (int p = 0; p < 17; p++) {
    snprintf(buf, sizeof buf, "%.*e", p, v);
    if (strtod(buf, nullptr) == v) break;
  }
  std::string s(buf);
  const bool neg = s[0] == '-';
  if (neg) s.erase(0, 1);
  const size_t e = s.find('e');
  const int exp = atoi(s.c_str() + e + 1);
  std::string digits;
  for (size_t i = 0; i < e; i++) if (s[i] != '.') digits += s[i];
  while (digits.size() > 1 && digits.back() == '0') digits.pop_back();
  const int point = exp + 1;  // digits before the decimal point
  std::string out;
  if (point <= 0) out = "0." + std::string((size_t)-point, '0') + digits;
  else if ((size_t)point >= digits.size()) out = digits + std::string((size_t)point - digits.size(), '0');
  else out = digits.substr(0, (size_t)point) + "." + digits.substr((size_t)point);
  return (neg ? "-" : "") + out;
}
// the type-tagged form of a composite key (tantivy's AfterKey): "str:…", "i64:…", "u64:…", "f64:…", "bool:…"
static std::string comp_key_tagged(const CompKey& k) {
  switch (k.t) {
    case CompKey::Bool: return k.u ? "bool:true" : "bool:false";
    case CompKey::Str: return "str:" + k.s;
    case CompKey::I64: return "i64:" + std::to_string(k.i);
    case CompKey::U64: return "u64:" + std::to_string(k.u);
    case CompKey::F64: return "f64:" + rust_display_f64(k.f);
    default: return "";
  }
}
static void opt_f64(bool some, double v, std::string& out) { if (some) json_f64(v, out); else out += "null"; }
static std::string range_num(double v) {
  std::string s;
  if (v == std::floor(v) && std::fabs(v) < 1e15) { char b[32]; snprintf(b, sizeof b, "%.0f", v); s = b; }
  else json_f64(v, s);
  return s;
}

static void fin_agg(const AggReq& req, const IAgg* a, std::string& out) {
  IAgg empty;
  empty.kind = (uint8_t)req.kind;
  if (!a) a = &empty;
  if (req.kind == AggReq::Percentiles) {
    // {"values": {"<percent>": value}} (keyed; the percent in Rust f64 Display form) or
    // {"values": [{"key": percent, "value": value}]}; an empty sketch gives null
    dds::Sketch s = a->sk;
    s.collapse();
    out += req.keyed ? "{\"values\":{" : "{\"values\":[";
    for (size_t i = 0; i < req.percents.size(); i++) {
      if (i) out += ",";
      double v = 0;
      const bool some = s.quantile(req.percents[i] / 100.0, &v);
      if (req.keyed) {
        json_escape(rust_display_f64(req.percents[i]), out);
        out += ":";
        opt_f64(some, v, out);
      } else {
        out += "{\"key\":";
        json_f64(req.percents[i], out);
        out += ",\"value\":";
        opt_f64(some, v, out);
        out += "}";
      }
    }
    out += req.keyed ? "}}" : "]}";
    return;
  }
  if (req.is_metric()) {
    bool some = a->m_count > 0;
    double avg = some ? a->m_sum / (double)a->m_count : 0;
    switch (req.kind) {
      case AggReq::Stats:
        out += "{\"avg\":"; opt_f64(some, avg, out);
        out += ",\"count\":" + std::to_string(a->m_count);
        out += ",\"max\":"; opt_f64(some, a->m_max, out);
        out += ",\"min\":"; opt_f64(some, a->m_min, out);
        out += ",\"sum\":"; json_f64(a->m_sum, out);
        out += "}";
        break;
      case AggReq::Avg: out += "{\"value\":"; opt_f64(some, avg, out); out += "}"; break;
      case AggReq::Sum: out += "{\"value\":"; json_f64(a->m_sum, out); out += "}"; break;
      case AggReq::Min: out += "{\"value\":"; opt_f64(some, a->m_min, out); out += "}"; break;
      case AggReq::Max: out += "{\"value\":"; opt_f64(some, a->m_max, out); out += "}"; break;
      default: out += "{\"value\":"; json_f64((double)a->m_count, out); out += "}"; break;
    }
    return;
  }
  auto subs = [&](const IBucket* b) {
    if (req.children.empty()) return;
    out += ",";
    std::string inner;
    fin_aggs(req.children, b ? &b->subs : nullptr, inner);
    out += inner.substr(1, inner.size() - 2);  // splice the members of {...}
  };
  if (req.kind == AggReq::Composite) {
    // {"after_key": {source: tagged key}, "buckets": [{"doc_count", "key": {source: key}, sub-aggregations}]};
    // after_key is the last bucket's key ({} without buckets), type-tagged so that it pages back exactly
    IAgg c;
    c.kind = a->kind;
    c.buckets = a->buckets;
    comp_sort_cut(req, c);
    auto plain = [&](const CompKey& k) {
      switch (k.t) {
        case CompKey::Null: out += "null"; break;
        case CompKey::Bool: out += k.u ? "true" : "false"; break;
        case CompKey::Str: json_escape(k.s, out); break;
        case CompKey::I64: out += std::to_string(k.i); break;
        case CompKey::U64: out += std::to_string(k.u); break;
        default: json_f64(k.f, out);
      }
    };
    out += "{\"after_key\":{";
    if (!c.buckets.empty()) {
      const std::vector<CompKey>& last = c.buckets.back().ckey;
      for (size_t i = 0; i < req.sources.size(); i++) {
        if (i) out += ",";
        json_escape(req.sources[i].name, out);
        out += ":";
        if (last[i].t == CompKey::Null) out += "null";
        else json_escape(comp_key_tagged(last[i]), out);
      }
    }
    out += "},\"buckets\":[";
    for (size_t bi = 0; bi < c.buckets.size(); bi++) {
      const IBucket& b = c.buckets[bi];
      if (bi) out += ",";
      out += "{\"doc_count\":" + std::to_string(b.count) + ",\"key\":{";
      for (size_t i = 0; i < req.sources.size(); i++) {
        if (i) out += ",";
        json_escape(req.sources[i].name, out);
        out += ":";
        plain(b.ckey[i]);
      }
      out += "}";
      subs(&b);
      out += "}";
    }
    out += "]}";
    return;
  }
  if (req.kind == AggReq::Terms) {
    uint64_t sum_other = a->sum_other;
    std::vector<const IBucket*> kept;
    for (uint32_t i : term_order(req, a->buckets)) {
      const IBucket& b = a->buckets[i];
      if (b.count < req.min_doc_count) continue;
      if (kept.size() < req.size) kept.push_back(&b);
      else sum_other += b.count;
    }
    out += "{\"buckets\":[";
    for (size_t i = 0; i < kept.size(); i++) {
      if (i) out += ",";
      out += "{\"doc_count\":" + std::to_string(kept[i]->count) + ",\"key\":";
      fin_key(kept[i]->key, out);
      subs(kept[i]);
      out += "}";
    }
    out += "],\"doc_count_error_upper_bound\":" + std::to_string(a->error_bound) + ",\"sum_other_doc_count\":" + std::to_string(sum_other) + "}";
    return;
  }
  if (req.kind == AggReq::Range) {
    // buckets in request order, plus the open-ended buckets needed to cover the whole axis
    struct RB { bool has_from, has_to; double from, to; std::string key; const IBucket* b; };
    std::vector<RB> rbs;
    for (size_t i = 0; i < req.ranges.size(); i++) {
      const IBucket* b = nullptr;
      for (auto& x : a->buckets) if ((size_t)x.hkey == i) b = &x;
      rbs.push_back({req.ranges[i].has_from, req.ranges[i].has_to, req.ranges[i].from, req.ranges[i].to, req.ranges[i].key, b});
    }
    out += "{\"buckets\":[";
    for (size_t i = 0; i < rbs.size(); i++) {
      if (i) out += ",";
      std::string key = rbs[i].key;
      if (key.empty()) key = (rbs[i].has_from ? range_num(rbs[i].from) : "*") + "-" + (rbs[i].has_to ? range_num(rbs[i].to) : "*");
      out += "{\"doc_count\":" + std::to_string(rbs[i].b ? rbs[i].b->count : 0);
      if (rbs[i].has_from) { out += ",\"from\":"; json_f64(rbs[i].from, out); }
      out += ",\"key\":";
      json_escape(key, out);
      if (rbs[i].has_to) { out += ",\"to\":"; json_f64(rbs[i].to, out); }
      subs(rbs[i].b);
      out += "}";
    }
    out += "]}";
    return;
  }
  // histogram / date_histogram: keys are in column units (ns for dates); output keys in request
  // units (ms for dates), gaps filled when min_doc_count == 0
  const double unit = a->is_date || req.kind == AggReq::DateHistogram ? 1e6 : 1.0;
  const double interval = req.interval * unit, offset = req.offset * unit;
  std::map<int64_t, const IBucket*> by_pos;
  for (auto& b : a->buckets) by_pos[(int64_t)std::llround((b.hkey - offset) / interval)] = &b;
  std::vector<std::pair<int64_t, const IBucket*>> seq;
  if (req.min_doc_count == 0) {
    bool any = !by_pos.empty();
    int64_t lo = any ? by_pos.begin()->first : 0, hi = any ? by_pos.rbegin()->first : -1;
    if (req.has_extended_bounds) {
      int64_t elo = (int64_t)qw_hist_pos(req.ext_min * unit, offset, interval), ehi = (int64_t)qw_hist_pos(req.ext_max * unit, offset, interval);
      if (elo <= ehi) {
        if (!any) { lo = elo; hi = ehi; any = true; }
        else { lo = std::min(lo, elo); hi = std::max(hi, ehi); }
      }
    }
    if (any) {
      if (hi - lo > 65000) fail(QWGPU_EINVALID_AGG, "aborting aggregation: too many histogram buckets (%lld)", (long long)(hi - lo + 1));
      for (int64_t p = lo; p <= hi; p++) {
        auto it = by_pos.find(p);
        seq.push_back({p, it == by_pos.end() ? nullptr : it->second});
      }
    }
  } else {
    for (auto& kv : by_pos) if (kv.second->count >= req.min_doc_count) seq.push_back(kv);
  }
  out += "{\"buckets\":[";
  bool first = true;
  for (auto& kv : seq) {
    double key = ((double)kv.first * interval + offset) / unit;
    if (req.has_hard_bounds && (key < req.hard_min || key > req.hard_max) && !kv.second) continue;
    if (!first) out += ",";
    first = false;
    out += "{\"doc_count\":" + std::to_string(kv.second ? kv.second->count : 0) + ",\"key\":";
    json_f64(key, out);
    if (req.kind == AggReq::DateHistogram) { out += ",\"key_as_string\":"; json_escape(rfc3339_from_ms(key), out); }
    subs(kv.second);
    out += "}";
  }
  out += "]}";
}

static void fin_aggs(const std::vector<AggReq>& reqs, const std::vector<IAgg>* aggs, std::string& out) {
  out += "{";
  for (size_t i = 0; i < reqs.size(); i++) {
    if (i) out += ",";
    json_escape(reqs[i].name, out);
    out += ":";
    fin_agg(reqs[i], aggs && i < aggs->size() ? &(*aggs)[i] : nullptr, out);
  }
  out += "}";
}

std::string finalize_aggs_json(const std::vector<AggReq>& reqs, const std::string& intermediate) {
  if (is_trace_ids_request(reqs)) {
    // the root passes the merged bytes through (root.rs:1111-1113); this is their human-readable serde form:
    // [{"trace_id": <32 hex digits>, "span_timestamp": <i64 ns>}, ...]
    static const char* hex = "0123456789abcdef";
    std::string out = "[";
    const std::vector<TraceSpan> v = intermediate.empty() ? std::vector<TraceSpan>() : decode_spans(intermediate);
    for (size_t i = 0; i < v.size(); i++) {
      if (i) out += ",";
      out += "{\"trace_id\":\"";
      for (int k = 0; k < 16; k++) { out += hex[v[i].id[k] >> 4]; out += hex[v[i].id[k] & 15]; }
      out += "\",\"span_timestamp\":" + std::to_string(v[i].ts) + "}";
    }
    return out + "]";
  }
  std::vector<IAgg> top;
  if (!intermediate.empty()) top = de_top(intermediate);
  if (!top.empty() && top.size() != reqs.size()) fail(QWGPU_EINTERNAL, "intermediate aggregation result does not match the request");
  std::string out;
  fin_aggs(reqs, top.empty() ? nullptr : &top, out);
  return out;
}

}  // namespace qw
