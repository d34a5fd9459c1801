// query_compile.cpp — (SearchRequest, doc mapper JSON, split directory) -> seam-C plan.
//
// Mirrors, for one split:
//   * DocMapper::query / build_query            quickwit-doc-mapper/src/query_builder.rs:158-236
//   * QueryAst -> TantivyQueryAst lowering       quickwit-query/src/query_ast/{mod.rs:230-270,
//       bool_query.rs, term_query.rs, full_text_query.rs:103-160, range_query.rs:141-205,
//       field_presence.rs, term_set_query.rs}
//   * TantivyBoolQuery::simplify                 quickwit-query/src/query_ast/tantivy_query_ast.rs:166-337
//   * filter = Must(ConstScoreQuery(q, 0.0))     tantivy_query_ast.rs:345-377
//   * rewrite_request (sort dropped when max_hits == 0; [start,end) timestamps folded into the AST)
//                                                quickwit-search/src/leaf.rs:712-729,841-946
//   * sort_by_from_request / make_collector_for_split   quickwit-search/src/collector.rs:994-1052
//   * SearchAfterSegment::new + convert_to_u64_ff_val   top_k_collector.rs:829-872, collector.rs:214-372
// Term dictionary lookups happen here, on the host, as they do in the reference (sstable lookup
// during warmup); only posting / column bytes are touched on the GPU.
#include <algorithm>
#include <cctype>
#include <climits>
#include <map>

#include "compile.h"
#include "ip_addr.h"
#include "regex.h"

namespace qw {

static const int64_t MIN_TIMESTAMP_SECONDS = 72057595;    // quickwit-datetime: 13 Apr 1972 23:59:55
static const int64_t MAX_TIMESTAMP_SECONDS = 8589934591;  // 16 Mar 2242 12:56:31

// quickwit_datetime::parse_timestamp (quickwit-datetime/src/date_time_parsing.rs:147-174)
static bool parse_timestamp_autodetect(int64_t ts, int64_t* nanos) {
  if (ts >= MIN_TIMESTAMP_SECONDS && ts <= MAX_TIMESTAMP_SECONDS) { *nanos = ts * 1000000000ll; return true; }
  if (ts >= MIN_TIMESTAMP_SECONDS * 1000 && ts <= MAX_TIMESTAMP_SECONDS * 1000) { *nanos = ts * 1000000ll; return true; }
  if (ts >= MIN_TIMESTAMP_SECONDS * 1000000 && ts <= MAX_TIMESTAMP_SECONDS * 1000000) { *nanos = ts * 1000ll; return true; }
  if (ts >= MIN_TIMESTAMP_SECONDS * 1000000000ll && ts <= MAX_TIMESTAMP_SECONDS * 1000000000ll) { *nanos = ts; return true; }
  return false;
}
static int64_t days_from_civil(int64_t y, unsigned m, unsigned d) {
  y -= m <= 2;
  const int64_t era = (y >= 0 ? y : y - 399) / 400;
  const unsigned yoe = (unsigned)(y - era * 400);
  const unsigned doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1;
  const unsigned doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
  return era * 146097 + (int64_t)doe - 719468;
}
// RFC 3339 / "%Y-%m-%d[ T]%H:%M:%S[.f]" / "%Y-%m-%d" (subset of json_literal.rs:24-39)
bool parse_datetime_str(const std::string& s, int64_t* nanos) {
  int y, mo, d, h = 0, mi = 0, se = 0, n = 0;
  if (sscanf(s.c_str(), "%4d-%2d-%2d%n", &y, &mo, &d, &n) != 3 || n != 10) {
    char* end = nullptr;
    long long v = strtoll(s.c_str(), &end, 10);
    if (end && *end == 0 && !s.empty()) return parse_timestamp_autodetect(v, nanos);
    return false;
  }
  const char* p = s.c_str() + 10;
  int64_t frac = 0, tz = 0;
  if (*p == 'T' || *p == 't' || *p == ' ') {
    int m2 = 0;
    if (sscanf(p + 1, "%2d:%2d:%2d%n", &h, &mi, &se, &m2) != 3) return false;
    p += 1 + m2;
    if (*p == '.') {
      p++;
      int digits = 0;
      while (isdigit((unsigned char)*p)) { if (digits < 9) { frac = frac * 10 + (*p - '0'); digits++; } p++; }
      while (digits++ < 9) frac *= 10;
    }
    if (*p == 'Z' || *p == 'z') p++;
    else if (*p == '+' || *p == '-') {
      int th, tm;
      if (sscanf(p + 1, "%2d:%2d", &th, &tm) != 2) return false;
      tz = (th * 3600 + tm * 60) * (*p == '-' ? -1 : 1);
      p += 6;
    }
  }
  if (*p) return false;
  int64_t secs = days_from_civil(y, (unsigned)mo, (unsigned)d) * 86400 + h * 3600 + mi * 60 + se - tz;
  *nanos = secs * 1000000000ll + frac;
  return true;
}

// tantivy "default" tokenizer, ASCII case folding (same rule as splitgen.tokenize_default)
std::vector<std::string> tokenize_text(const std::string& text, uint32_t tokenizer) {
  std::vector<std::string> out;
  if (tokenizer == QW_TOK_RAW) { out.push_back(text); return out; }
  std::string cur;
  for (unsigned char c : text) {
    if (isalnum(c) || c >= 0x80) cur += (char)(c < 0x80 ? tolower(c) : c);
    else if (!cur.empty()) { if (cur.size() <= 255) out.push_back(cur); cur.clear(); }
  }
  if (!cur.empty() && cur.size() <= 255) out.push_back(cur);
  return out;
}

DocMapperInfo parse_doc_mapper(const std::string& json) {
  DocMapperInfo dm;
  if (json.empty()) return dm;
  Json j = parse_json(json, QWGPU_EINVALID_ARG);
  const Json* root = &j;
  if (const Json* inner = j.get("doc_mapping")) root = inner;  // tolerate an index-config wrapper
  dm.timestamp_field = root->str_or("timestamp_field", "");
  if (const Json* fm = root->get("field_mappings"))
    for (auto& f : fm->arr) {
      DocMapperInfo::Field fi;
      fi.name = f.str_or("name", "");
      fi.type = f.str_or("type", "text");
      fi.tokenizer = f.str_or("tokenizer", "default");
      fi.fast_precision = f.str_or("fast_precision", "seconds");
      fi.indexed = f.bool_or("indexed", true);
      dm.fields.push_back(fi);
    }
  if (const Json* d = root->get("default_search_fields"))
    for (auto& f : d->arr) if (f.is_str()) dm.default_search_fields.push_back(f.s);
  return dm;
}

static int64_t precision_ns(const DocMapperInfo& dm, const std::string& field) {
  for (auto& f : dm.fields)
    if (f.name == field) {
      if (f.fast_precision == "milliseconds") return 1000000;
      if (f.fast_precision == "microseconds") return 1000;
      if (f.fast_precision == "nanoseconds") return 1;
      return 1000000000;
    }
  return 1000000000;
}
static int64_t truncate_ns(int64_t ns, int64_t prec) {  // DateTime::truncate
  int64_t r = ns % prec;
  if (r < 0) r += prec;
  return ns - r;
}

// ---- TantivyQueryAst mirror ------------------------------------------------------------------------
struct TQ {
  enum Kind { Bool, Term, Range, Exists, All, None, Phrase, PhrasePrefix, TermSet, ColSet, Cache } kind = None;  // Cache: must[0]
  std::vector<uint32_t> phrase_terms;  // Phrase / PhrasePrefix: (exact) term ords in phrase order (offset k = position k)
  std::vector<uint32_t> prefix_terms;  // PhrasePrefix: the expansions of the last slot (offset = phrase_terms.size());
                                       // TermSet: the term ords of one field, ascending
  std::vector<uint64_t> set_values;    // ColSet: the values of `column` (mapped-u64 space), ascending
  int group = -1;  // a leaf of a set group (set_groups_to_nodes): the group's number, in query order
  bool opaque = false;  // wrapped in a BoostQuery leaf: not subject to bool flattening / const folding
  std::vector<TQ> must, must_not, should, filter;
  bool has_msm = false;
  size_t msm = 0;
  float boost = 1.0f;
  uint32_t term_ord = 0xFFFFFFFFu;
  uint32_t column = 0xFFFFFFFFu;
  uint64_t lo = 0, hi = 0;
  int const_pred() const { return opaque ? -1 : (kind == All ? 1 : (kind == None ? 0 : -1)); }  // 1 all, 0 none
};
static TQ tq_all() { TQ t; t.kind = TQ::All; return t; }
static TQ tq_none() { TQ t; t.kind = TQ::None; return t; }

// remove_with_guard (tantivy_query_ast.rs:141-156)
static void remove_with_guard(std::vector<TQ>& v, int to_remove, bool stop_before_empty) {
  size_t i = 0;
  while (i < v.size()) {
    if (stop_before_empty && v.size() == 1) break;
    if (v[i].const_pred() == to_remove) { std::swap(v[i], v.back()); v.pop_back(); }
    else i++;
  }
}

// TantivyBoolQuery::simplify (tantivy_query_ast.rs:190-337)
static TQ simplify(TQ q) {
  if (q.kind != TQ::Bool || q.opaque) return q;
  for (auto* vec : {&q.must, &q.should, &q.must_not, &q.filter})
    for (auto& c : *vec) c = simplify(std::move(c));
  for (auto* vec : {&q.must, &q.filter})
    for (auto& c : *vec) if (c.const_pred() == 0) return tq_none();
  if (q.should.empty() && q.must.empty() && q.filter.empty() && q.must_not.empty() && (!q.has_msm || q.msm == 0)) return tq_all();
  auto is_plain_bool = [](const TQ& t) { return t.kind == TQ::Bool && !t.opaque; };
  std::vector<TQ> new_must;
  for (auto& m : q.must) {
    if (is_plain_bool(m) && m.should.empty() && !m.has_msm) {
      for (auto& c : m.must) new_must.push_back(std::move(c));
      for (auto& c : m.filter) q.filter.push_back(std::move(c));
      for (auto& c : m.must_not) q.must_not.push_back(std::move(c));
    } else new_must.push_back(std::move(m));
  }
  q.must = std::move(new_must);
  std::vector<TQ> new_filter;
  for (auto& f : q.filter) {
    if (is_plain_bool(f) && f.should.empty() && !f.has_msm) {
      for (auto& c : f.must) new_filter.push_back(std::move(c));
      for (auto& c : f.filter) new_filter.push_back(std::move(c));
      for (auto& c : f.must_not) q.must_not.push_back(std::move(c));
    } else new_filter.push_back(std::move(f));
  }
  q.filter = std::move(new_filter);
  if (!q.has_msm) {
    std::vector<TQ> new_should;
    for (auto& s : q.should) {
      if (is_plain_bool(s) && s.must.empty() && s.filter.empty() && s.must_not.empty() && !s.has_msm)
        for (auto& c : s.should) new_should.push_back(std::move(c));
      else new_should.push_back(std::move(s));
    }
    q.should = std::move(new_should);
  }
  remove_with_guard(q.must, 1, true);
  bool no_positive = q.must.empty();
  remove_with_guard(q.filter, 1, no_positive);
  no_positive = no_positive && q.filter.empty();
  if (!q.filter.empty()) remove_with_guard(q.must, 1, false);
  remove_with_guard(q.should, 0, no_positive);
  no_positive = no_positive && q.should.empty();
  remove_with_guard(q.must_not, 0, no_positive);
  for (auto* vec : {&q.must, &q.filter})
    for (auto& c : *vec) if (c.const_pred() == 0) return tq_none();
  for (auto& c : q.must_not) if (c.const_pred() == 1) return tq_none();
  bool has_positive = !(q.must.empty() && q.should.empty() && q.filter.empty());
  if (!has_positive) {
    if (q.has_msm && q.msm > 0) return tq_none();
    bool all_none = true;
    for (auto& c : q.must_not) if (c.const_pred() != 0) all_none = false;
    if (all_none) return tq_all();
    q.must.push_back(tq_all());
  } else {
    size_t n = q.must.size() + q.should.size() + q.must_not.size() + q.filter.size();
    if (n == 1 && !q.has_msm) {
      if (!q.must.empty()) return std::move(q.must[0]);
      if (!q.should.empty()) return std::move(q.should[0]);
    }
  }
  return q;
}

static void apply_boost(TQ& q, float b) {
  q.boost *= b;
  for (auto* vec : {&q.must, &q.should, &q.must_not, &q.filter})
    for (auto& c : *vec) apply_boost(c, b);
}

// ---- literal interpretation (quickwit-query/src/json_literal.rs) -----------------------------------
static bool lit_u64(const Json& v, uint64_t* out) {
  if (v.type == Json::U64) { *out = v.u; return true; }
  if (v.type == Json::I64) { if (v.i < 0) return false; *out = (uint64_t)v.i; return true; }
  if (v.type == Json::Str) { char* e; errno = 0; unsigned long long x = strtoull(v.s.c_str(), &e, 10); if (errno || *e || v.s.empty() || v.s[0] == '-') return false; *out = x; return true; }
  return false;
}
static bool lit_i64(const Json& v, int64_t* out) {
  if (v.type == Json::I64) { *out = v.i; return true; }
  if (v.type == Json::U64) { if (v.u > (uint64_t)INT64_MAX) return false; *out = (int64_t)v.u; return true; }
  if (v.type == Json::Str) { char* e; errno = 0; long long x = strtoll(v.s.c_str(), &e, 10); if (errno || *e || v.s.empty()) return false; *out = x; return true; }
  return false;
}
static bool lit_f64(const Json& v, double* out) {
  if (v.is_num()) { *out = v.as_f64(); return true; }
  if (v.type == Json::Str) { char* e; double x = strtod(v.s.c_str(), &e); if (*e || v.s.empty()) return false; *out = x; return true; }
  return false;
}
static bool lit_datetime(const Json& v, int64_t* nanos) {
  if (v.type == Json::Str) return parse_datetime_str(v.s, nanos);
  int64_t i;
  if (lit_i64(v, &i) && v.type != Json::F64) return parse_timestamp_autodetect(i, nanos);
  return false;
}
static std::string lit_str(const Json& v) {
  if (v.type == Json::Str) return v.s;
  if (v.type == Json::Bool) return v.b ? "true" : "false";
  std::string s;
  if (v.type == Json::U64) s = std::to_string(v.u);
  else if (v.type == Json::I64) s = std::to_string(v.i);
  else if (v.type == Json::F64) json_f64(v.f, s);
  return s;
}

// value of a typed column in mapped-u64 space; false when the literal does not fit the type
static bool literal_to_mapped(const QwImgColumn& c, const Json& v, const DocMapperInfo& dm, const std::string& field, uint64_t* out) {
  switch (c.type) {
    case QW_COL_U64: return lit_u64(v, out);
    case QW_COL_I64: { int64_t i; if (!lit_i64(v, &i)) return false; *out = i64_to_u64(i); return true; }
    case QW_COL_F64: { double d; if (!lit_f64(v, &d)) return false; *out = f64_to_u64(d); return true; }
    case QW_COL_BOOL: {
      if (v.type == Json::Bool) { *out = v.b; return true; }
      if (v.type == Json::Str && (v.s == "true" || v.s == "false")) { *out = v.s == "true"; return true; }
      return false;
    }
    case QW_COL_DATETIME: { int64_t ns; if (!lit_datetime(v, &ns)) return false; *out = i64_to_u64(truncate_ns(ns, precision_ns(dm, field))); return true; }
    default: return false;
  }
}
static const char* col_type_name(uint32_t t) {
  static const char* n[] = {"u64", "i64", "f64", "bool", "datetime", "text", "bytes", "ip"};
  return t < 8 ? n[t] : "?";
}

struct Ctx {
  const ImageView& img;
  const DocMapperInfo& dm;
  bool scoring = false;             // the request ranks by _score
  mutable int unscored_depth = 0;   // > 0 while building a must_not / filter subtree (its scores are never read)
  mutable int groups = 0;           // set groups numbered so far
};

// Constant-score set queries (TermSetQuery, wildcard -> AutomatonWeight): tantivy gives every matching document the
// score 1.0 (ConstScorer over a bitset). The plan has no constant-score node, so these compile to an unscored filter —
// exact for every sort except BM25 ranking with the node in a scoring position, which is refused instead of ranked
// differently.
static void refuse_const_score_under_ranking(const Ctx& cx, const char* what) {
  if (cx.scoring && cx.unscored_depth == 0)
    fail(QWGPU_EUNSUPPORTED, "`%s` in a scoring clause of a query ranked by _score is not implemented on the GPU path (constant score 1.0)", what);
}

// ---- wildcard queries (quickwit-query/src/query_ast/wildcard_query.rs) ------------------------------------------
struct GlobPart { int kind; std::string text; };  // 0 = text, 1 = `*`, 2 = `?`
// parse_wildcard_query (wildcard_query.rs:43-72): `*`, `?`, backslash escapes the next character
static std::vector<GlobPart> parse_wildcard(const std::string& q) {
  std::vector<GlobPart> out;
  auto text = [&](const std::string& t) { if (!out.empty() && out.back().kind == 0) out.back().text += t; else out.push_back({0, t}); };
  size_t i = 0;
  auto utf8_len = [](unsigned char c) { return c < 0x80 ? 1u : (c >> 5) == 6 ? 2u : (c >> 4) == 14 ? 3u : (c >> 3) == 30 ? 4u : 1u; };
  while (i < q.size()) {
    const char c = q[i];
    if (c == '*') { out.push_back({1, ""}); i++; }
    else if (c == '?') { out.push_back({2, ""}); i++; }
    else if (c == '\\') {
      if (i + 1 >= q.size()) break;  // a trailing escape is dropped
      const size_t n = std::min<size_t>(utf8_len((unsigned char)q[i + 1]), q.size() - i - 1);
      text(q.substr(i + 1, n));
      i += 1 + n;
    } else { text(std::string(1, c)); i++; }
  }
  return out;
}
static bool glob_match(const std::vector<GlobPart>& parts, size_t pi, const uint8_t* s, size_t n, size_t si) {
  auto cp_len = [&](size_t at) { const unsigned char c = s[at]; size_t l = c < 0x80 ? 1 : (c >> 5) == 6 ? 2 : (c >> 4) == 14 ? 3 : (c >> 3) == 30 ? 4 : 1; return std::min(l, n - at); };
  for (; pi < parts.size(); pi++) {
    const GlobPart& p = parts[pi];
    if (p.kind == 0) {
      if (n - si < p.text.size() || memcmp(s + si, p.text.data(), p.text.size()) != 0) return false;
      si += p.text.size();
    } else if (p.kind == 2) {
      if (si >= n) return false;
      si += cp_len(si);
    } else {
      // `.*`: every suffix that starts on a code point boundary
      for (size_t k = si;; k += cp_len(k)) {
        if (glob_match(parts, pi + 1, s, n, k)) return true;
        if (k >= n) return false;
      }
    }
  }
  return si == n;
}

static TQ term_leaf(const Ctx& cx, uint32_t field, const std::string& token) {
  TQ t;
  t.kind = TQ::Term;
  int ord = cx.img.find_term(field, (const uint8_t*)token.data(), (uint32_t)token.size());
  t.term_ord = ord < 0 ? 0xFFFFFFFFu : (uint32_t)ord;
  return t;
}
// ---- phrase prefix queries (quickwit-query/src/query_ast/phrase_prefix_query.rs, tantivy PhrasePrefixQuery) -----

// Tokenizer named by a phrase_prefix / bool_prefix query (FullTextParams::text_analyzer): the image applies `raw` and
// `default`; the other analyzers quickwit registers (tokenizers/mod.rs) are refused, any other name is an error.
static uint32_t prefix_query_tokenizer(const std::string& name, uint32_t field_tokenizer) {
  if (name.empty()) return field_tokenizer;
  if (name == "raw") return QW_TOK_RAW;
  if (name == "default") return QW_TOK_DEFAULT;
  static const char* registered[] = {"raw_lowercase", "lowercase", "whitespace", "chinese_compatible", "source_code_default", "source_code_with_hex"};
  for (const char* r : registered)
    if (name == r) fail(QWGPU_EUNSUPPORTED, "tokenizer `%s` is not implemented on the GPU path", name.c_str());
  fail(QWGPU_EINVALID_QUERY, "invalid query: no tokenizer named `%s` is registered", name.c_str());
}

// The prefix's expansions in one split: the field's first `max_expansions` terms, in byte order, that start with
// `prefix` (the TermRange [prefix, prefix_end) with limit max_expansions of query_builder.rs)
static std::vector<uint32_t> expand_prefix(const ImageView& img, uint32_t field, const std::string& prefix, uint64_t max_expansions) {
  const QwImgField& F = img.fields[field];
  auto less = [&](uint32_t t) {  // term t < prefix
    const QwImgTerm& T = img.terms[t];
    const uint32_t m = std::min<uint32_t>(T.bytes_len, (uint32_t)prefix.size());
    const int c = memcmp(img.term_bytes + T.bytes_off, prefix.data(), m);
    return c < 0 || (c == 0 && T.bytes_len < prefix.size());
  };
  uint32_t lo = F.first_term, hi = F.first_term + F.num_terms;
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo) / 2;
    if (less(mid)) lo = mid + 1; else hi = mid;
  }
  std::vector<uint32_t> out;
  for (uint32_t t = lo; t < F.first_term + F.num_terms && out.size() < max_expansions; t++) {
    const QwImgTerm& T = img.terms[t];
    if (T.bytes_len < prefix.size() || memcmp(img.term_bytes + T.bytes_off, prefix.data(), prefix.size()) != 0) break;
    out.push_back(t);
  }
  return out;
}

// PhrasePrefixQuery::new_with_offset(tokens) with max_expansions, on a text field of the split. One token: a doc
// matches when it holds any expansion (tantivy's range query with a limit) — an unscored set filter of TERM nodes,
// the wildcard shape. More tokens: QW_NODE_PHRASE_PREFIX. Both are constant-score in tantivy's sense only as far as
// the visible sources go, so neither is served in a scoring clause under _score ranking.
static TQ phrase_prefix_leaf(const Ctx& cx, uint32_t f, const std::vector<std::string>& tokens, uint64_t max_expansions) {
  if (tokens.size() > 1 && !(cx.img.fields[f].flags & QW_FIELD_HAS_POSITIONS))
    fail(QWGPU_EINVALID_QUERY, "invalid query: trying to run a phrase prefix query on a field which does not have positions indexed");
  if (tokens.size() > QW_MAX_PHRASE_TERMS)
    fail(QWGPU_EUNSUPPORTED, "phrase prefixes of more than %d terms are not implemented on the GPU path", QW_MAX_PHRASE_TERMS);
  refuse_const_score_under_ranking(cx, "phrase_prefix");
  TQ ph;
  ph.kind = TQ::PhrasePrefix;
  for (size_t i = 0; i + 1 < tokens.size(); i++) {
    const int ord = cx.img.find_term(f, (const uint8_t*)tokens[i].data(), (uint32_t)tokens[i].size());
    if (ord < 0) return tq_none();  // a split without one of the exact terms matches nothing
    ph.phrase_terms.push_back((uint32_t)ord);
  }
  ph.prefix_terms = expand_prefix(cx.img, f, tokens.back(), max_expansions);
  if (ph.prefix_terms.empty()) return tq_none();
  if (tokens.size() > 1) return ph;
  TQ b;
  b.kind = TQ::Bool;
  const int group = cx.groups++;
  for (uint32_t t : ph.prefix_terms) {
    TQ leaf;
    leaf.kind = TQ::Term;
    leaf.term_ord = t;
    leaf.group = group;
    b.should.push_back(std::move(leaf));
  }
  TQ outer;
  outer.kind = TQ::Bool;
  outer.filter.push_back(std::move(b));
  return outer;
}

// RegexQuery::to_resolved + build_tantivy_ast_impl (regex_query.rs): the field must be an indexed text field; a
// tokenizer that lowercases prefixes `(?i)` unless the pattern's leading flags already hold an `i`. The pattern is
// parsed before the split's terms are looked at, so a bad pattern fails on every split. The matching terms become one
// TERM_SET node: tantivy's AutomatonWeight is constant-score, so it is served wherever its score is not read.
static TQ regex_leaf(const Ctx& cx, const std::string& field, const std::string& regex) {
  const int f = cx.img.find_field(field);
  const DocMapperInfo::Field* fd = nullptr;
  for (auto& d : cx.dm.fields) if (d.name == field) fd = &d;
  const int c = cx.img.find_column(field);
  if ((f >= 0 && cx.img.fields[f].tokenizer == QW_TOK_IP) || (c >= 0 && cx.img.columns[c].type == QW_COL_IP))
    fail(QWGPU_EINVALID_QUERY, "invalid query: trying to run a regex query on a non-text field");
  if (f < 0) {
    if ((c >= 0 && cx.img.columns[c].type != QW_COL_STR) || (fd && fd->type != "text" && fd->type != "json"))
      fail(QWGPU_EINVALID_QUERY, "invalid query: trying to run a regex query on a non-text field");
    if (c >= 0 || (fd && !fd->indexed)) fail(QWGPU_EINVALID_QUERY, "invalid query: field %s is not full-text searchable", field.c_str());
    if (!fd) fail(QWGPU_EINVALID_QUERY, "invalid query: field does not exist: `%s`", field.c_str());
  }
  const bool lowercases = f >= 0 ? cx.img.fields[f].tokenizer != QW_TOK_RAW : fd->tokenizer != "raw";
  rx::Regex re(lowercases && !rx::has_case_insensitive_flag(regex) ? "(?i)" + regex : regex);
  if (f < 0) return tq_none();  // declared in the doc mapping but without a single term in this split
  refuse_const_score_under_ranking(cx, "regex");
  TQ t;
  t.kind = TQ::TermSet;
  t.prefix_terms = re.matching_terms(cx.img, (uint32_t)f);
  if (t.prefix_terms.empty()) return tq_none();
  if (t.prefix_terms.size() > QW_MAX_SET_TERMS)
    fail(QWGPU_EUNSUPPORTED, "regex with %zu expansions in split (the GPU path takes at most %d)", t.prefix_terms.size(), QW_MAX_SET_TERMS);
  return t;
}

static TQ range_leaf(uint32_t column, uint64_t lo, uint64_t hi) {
  TQ t;
  t.kind = TQ::Range;
  t.column = column;
  t.lo = lo;
  t.hi = hi;
  return t;
}

// ---- `ip` fields (json_literal.rs:135-140, query_ast/utils.rs:174-178) ----------------------------------------------
// A fast `ip` field is a QW_COL_IP column, an indexed one a field of 16-byte terms (QW_TOK_IP); a field of neither kind
// in this split is an `ip` field when the doc mapping declares it so.
static bool is_ip_field(const Ctx& cx, const std::string& field) {
  const int c = cx.img.find_column(field);
  if (c >= 0) return cx.img.columns[c].type == QW_COL_IP;
  const int f = cx.img.find_field(field);
  if (f >= 0) return cx.img.fields[f].tokenizer == QW_TOK_IP;
  for (auto& fd : cx.dm.fields) if (fd.name == field) return fd.type == "ip";
  return false;
}
static std::string ip_literal(const std::string& field, const std::string& text) {
  uint8_t a[16];
  if (!parse_ip_addr(text, a))
    fail(QWGPU_EINVALID_QUERY, "invalid query: expected a `ip` search value for field `%s`, got `%s`", field.c_str(), text.c_str());
  return std::string((const char*)a, 16);
}
// TermQuery on an `ip` field: the whole text is one address, never tokenized. On a fast field an equality on the
// ordinal (the dictionary is sorted, so an address present in the split has exactly one), else a posting lookup of
// the 16-byte term. Both run unscored: a scoring clause under _score ranking is refused.
static TQ ip_term(const Ctx& cx, const std::string& field, const std::string& text) {
  const std::string addr = ip_literal(field, text);
  refuse_const_score_under_ranking(cx, "ip term");
  const int c = cx.img.find_column(field);
  if (c >= 0) {
    bool exact;
    const uint32_t ord = cx.img.dict_lower_bound(cx.img.columns[c], (const uint8_t*)addr.data(), 16, &exact);
    return exact ? range_leaf((uint32_t)c, ord, ord) : tq_none();
  }
  const int f = cx.img.find_field(field);
  return f >= 0 ? term_leaf(cx, (uint32_t)f, addr) : tq_none();
}

// full_text_query / FullTextParams::make_query (full_text_query.rs:103-160, utils.rs:73-200)
static TQ full_text(const Ctx& cx, const std::string& field, const std::string& text, const std::string& tokenizer_override,
                    const std::string& mode, bool op_and, int zero_terms_all, bool lenient, uint32_t slop = 0,
                    uint64_t max_expansions = 50) {
  if (is_ip_field(cx, field)) return ip_term(cx, field, text);
  int f = cx.img.find_field(field);
  if (f < 0) {
    int c = cx.img.find_column(field);
    if (c >= 0 && cx.img.columns[c].type == QW_COL_BYTES)
      fail(QWGPU_EUNSUPPORTED, "queries on bytes field `%s` are not supported on the GPU path", field.c_str());
    if (c >= 0 && cx.img.columns[c].type != QW_COL_STR) {
      // numeric / bool / datetime field: TermQuery on the typed value == column equality
      Json lit; lit.type = Json::Str; lit.s = text;
      uint64_t m;
      if (!literal_to_mapped(cx.img.columns[c], lit, cx.dm, field, &m))
        fail(QWGPU_EINVALID_QUERY, "invalid query: expected a `%s` search value for field `%s`, got `%s`", col_type_name(cx.img.columns[c].type), field.c_str(), text.c_str());
      return range_leaf((uint32_t)c, m, m);
    }
    if (c >= 0) {  // fast-only raw text: equality on the ordinal
      bool exact;
      uint32_t ord = cx.img.dict_lower_bound(cx.img.columns[c], (const uint8_t*)text.data(), (uint32_t)text.size(), &exact);
      return exact ? range_leaf((uint32_t)c, ord, ord) : tq_none();
    }
    bool known = false;
    for (auto& fd : cx.dm.fields) if (fd.name == field) known = true;
    if (lenient || known) return tq_none();  // declared in the doc mapping but empty in this split
    fail(QWGPU_EINVALID_QUERY, "invalid query: field does not exist: `%s`", field.c_str());
  }
  uint32_t tok = cx.img.fields[f].tokenizer;
  if (mode == "bool_prefix") tok = prefix_query_tokenizer(tokenizer_override, tok);
  else if (!tokenizer_override.empty()) tok = tokenizer_override == "raw" ? QW_TOK_RAW : QW_TOK_DEFAULT;
  std::vector<std::string> tokens = tokenize_text(text, tok);
  if (tokens.empty()) return zero_terms_all ? tq_all() : tq_none();
  if (tokens.size() == 1) return term_leaf(cx, (uint32_t)f, tokens[0]);
  bool has_positions = (cx.img.fields[f].flags & QW_FIELD_HAS_POSITIONS) != 0;
  if (mode == "phrase" || (mode == "phrase_fallback_to_intersection" && has_positions)) {
    if (!has_positions)
      fail(QWGPU_EINVALID_QUERY, "invalid query: Applied phrase query on field which does not have positions indexed");
    if (slop != 0) fail(QWGPU_EUNSUPPORTED, "phrase queries with slop > 0 are not implemented on the GPU path yet");
    if (tokens.size() > QW_MAX_PHRASE_LEN) fail(QWGPU_EUNSUPPORTED, "phrases of more than %d terms are not implemented on the GPU path", QW_MAX_PHRASE_LEN);
    // TantivyPhraseQuery::new_with_offset(terms) (full_text_query.rs:140-156): a term missing from the split
    // means no doc can match
    TQ ph;
    ph.kind = TQ::Phrase;
    for (auto& t : tokens) {
      int ord = cx.img.find_term((uint32_t)f, (const uint8_t*)t.data(), (uint32_t)t.size());
      if (ord < 0) return tq_none();
      ph.phrase_terms.push_back((uint32_t)ord);
    }
    return ph;
  }
  if (mode == "bool_prefix") {
    // FullTextMode::BoolPrefix (full_text_query.rs:124-139): every token but the last is a term query, the last a
    // one-token phrase prefix; clauses joined by the operator
    TQ b;
    b.kind = TQ::Bool;
    std::vector<TQ>& clauses = op_and ? b.must : b.should;
    for (size_t i = 0; i + 1 < tokens.size(); i++) clauses.push_back(term_leaf(cx, (uint32_t)f, tokens[i]));
    clauses.push_back(phrase_prefix_leaf(cx, (uint32_t)f, {tokens.back()}, max_expansions));
    return b;
  }
  TQ b;
  b.kind = TQ::Bool;
  bool conj = mode == "phrase_fallback_to_intersection" ? true : op_and;
  for (auto& t : tokens) (conj ? b.must : b.should).push_back(term_leaf(cx, (uint32_t)f, t));
  return b;
}

static bool bound_of(const Json& b, const Json** val, bool* included) {
  if (b.is_str()) { if (b.s == "Unbounded") return false; fail(QWGPU_EINVALID_QUERY, "invalid query: bad range bound"); }
  if (const Json* v = b.get("Included")) { *val = v; *included = true; return true; }
  if (const Json* v = b.get("Excluded")) { *val = v; *included = false; return true; }
  fail(QWGPU_EINVALID_QUERY, "invalid query: bad range bound");
}

// RangeQuery::build_tantivy_ast_impl (range_query.rs:141-205) -> FastFieldRangeQuery
static TQ range_query(const Ctx& cx, const std::string& field, const Json* lower, const Json* upper) {
  int c = cx.img.find_column(field);
  if (c < 0) {
    bool known = cx.img.find_field(field) >= 0;
    for (auto& fd : cx.dm.fields) if (fd.name == field) known = true;
    if (!known) fail(QWGPU_EINVALID_QUERY, "invalid query: field does not exist: `%s`", field.c_str());
    if (cx.img.find_field(field) >= 0)
      fail(QWGPU_EINVALID_QUERY, "invalid query: range queries are only supported for fast fields. (`%s` is not a fast field)", field.c_str());
    return tq_none();  // fast field with no value in this split
  }
  const QwImgColumn& col = cx.img.columns[c];
  if (col.type == QW_COL_BYTES) fail(QWGPU_EUNSUPPORTED, "range queries on bytes field `%s` are not supported on the GPU path", field.c_str());
  if (col.type == QW_COL_BOOL) fail(QWGPU_EINVALID_QUERY, "invalid query: range queries are not supported for field `%s` of type `bool`", field.c_str());
  uint64_t lo = 0, hi = ~0ull;
  const Json* v;
  bool inc;
  auto conv = [&](const Json& lit, bool is_lower, bool included) -> bool {  // false => empty range
    uint64_t m;
    if (col.type == QW_COL_STR || col.type == QW_COL_IP) {
      // an address bound becomes an ordinal bound through the split's sorted dictionary, as a string bound does
      std::string s = col.type == QW_COL_IP ? ip_literal(field, lit_str(lit)) : lit_str(lit);
      bool exact;
      uint32_t lb = cx.img.dict_lower_bound(col, (const uint8_t*)s.data(), (uint32_t)s.size(), &exact);
      if (is_lower) { lo = (exact && !included) ? lb + 1 : lb; return true; }
      if (exact && included) { hi = lb; return true; }
      if (lb == 0) return false;
      hi = lb - 1;
      return true;
    }
    if (!literal_to_mapped(col, lit, cx.dm, field, &m))
      fail(QWGPU_EINVALID_QUERY, "invalid query: expected a `%s` boundary for field `%s`", col_type_name(col.type), field.c_str());
    if (is_lower) { if (!included) { if (m == ~0ull) return false; m++; } lo = m; }
    else { if (!included) { if (m == 0) return false; m--; } hi = m; }
    return true;
  };
  if (lower && bound_of(*lower, &v, &inc) && !conv(*v, true, inc)) return tq_none();
  if (upper && bound_of(*upper, &v, &inc) && !conv(*v, false, inc)) return tq_none();
  if (lo > hi) return tq_none();
  return range_leaf((uint32_t)c, lo, hi);
}

static TQ build(const Ctx& cx, const Json& q, int depth);

static std::vector<TQ> build_list(const Ctx& cx, const Json* arr, int depth) {
  std::vector<TQ> out;
  if (arr) for (auto& c : arr->arr) out.push_back(build(cx, c, depth + 1));
  return out;
}

static TQ build(const Ctx& cx, const Json& q, int depth) {
  if (depth > 32) fail(QWGPU_EINVALID_QUERY, "invalid query: nesting too deep");
  if (q.is_str()) {  // unit variants serialise as {"type": "..."} but tolerate bare strings
    if (q.s == "match_all") return tq_all();
    if (q.s == "match_none") return tq_none();
  }
  std::string type = q.str_or("type", "");
  if (type == "match_all") return tq_all();
  if (type == "match_none") return tq_none();
  if (type == "bool") {
    TQ b;
    b.kind = TQ::Bool;
    b.must = build_list(cx, q.get("must"), depth);
    b.should = build_list(cx, q.get("should"), depth);
    cx.unscored_depth++;
    b.must_not = build_list(cx, q.get("must_not"), depth);
    b.filter = build_list(cx, q.get("filter"), depth);
    cx.unscored_depth--;
    if (const Json* m = q.get("minimum_should_match")) if (m->is_num()) { b.has_msm = true; b.msm = (size_t)m->as_f64(); }
    return b;
  }
  if (type == "term") return full_text(cx, q.str_or("field", ""), q.str_or("value", ""), "raw", "bool", false, 0, false);
  if (type == "full_text") {
    const Json* params = q.get("params");
    std::string tok, mode = "bool";
    bool op_and = false;
    int zero_all = 0;
    uint32_t slop = 0;
    uint64_t max_expansions = 50;
    if (params) {
      tok = params->str_or("tokenizer", "");
      if (const Json* m = params->get("mode")) {
        mode = m->str_or("type", "bool");
        if (const Json* sl = m->get("slop")) slop = (uint32_t)sl->as_f64();
        if (const Json* me = m->get("max_expansions")) if (me->is_num()) max_expansions = (uint64_t)me->as_f64();
        std::string op = m->str_or("operator", "Or");
        op_and = op == "And" || op == "AND" || op == "and";
      }
      zero_all = params->str_or("zero_terms_query", "none") == "all";
    }
    return full_text(cx, q.str_or("field", ""), q.str_or("text", ""), tok, mode, op_and, zero_all, q.bool_or("lenient", false), slop, max_expansions);
  }
  if (type == "phrase_prefix") {
    // PhrasePrefixQuery::build_tantivy_ast_impl (phrase_prefix_query.rs): `lenient` covers a missing field only
    const std::string field = q.str_or("field", ""), phrase = q.str_or("phrase", "");
    uint64_t max_expansions = 50;
    if (const Json* me = q.get("max_expansions")) if (me->is_num()) max_expansions = (uint64_t)me->as_f64();
    const Json* params = q.get("params");
    const std::string tok_name = params ? params->str_or("tokenizer", "") : "";
    const bool zero_all = params && params->str_or("zero_terms_query", "none") == "all";
    const int f = cx.img.find_field(field);
    if (is_ip_field(cx, field)) fail(QWGPU_EINVALID_QUERY, "invalid query: trying to run a PhrasePrefix query on a non-text field");
    if (f < 0) {
      const int c = cx.img.find_column(field);
      bool known = false, text = true;
      uint32_t field_tok = QW_TOK_DEFAULT;
      for (auto& fd : cx.dm.fields)
        if (fd.name == field) { known = true; text = fd.type == "text" || fd.type == "json"; field_tok = fd.tokenizer == "raw" ? QW_TOK_RAW : QW_TOK_DEFAULT; }
      if ((c >= 0 && cx.img.columns[c].type != QW_COL_STR) || !text)
        fail(QWGPU_EINVALID_QUERY, "invalid query: trying to run a PhrasePrefix query on a non-text field");
      if (!known && !q.bool_or("lenient", false)) fail(QWGPU_EINVALID_QUERY, "invalid query: field does not exist: `%s`", field.c_str());
      if (!known) return tq_none();
      // declared in the doc mapping but without a single term in this split: no expansion can exist
      const uint32_t tok = prefix_query_tokenizer(tok_name, field_tok);
      return zero_all && tokenize_text(phrase, tok).empty() ? tq_all() : tq_none();
    }
    const uint32_t tok = prefix_query_tokenizer(tok_name, cx.img.fields[f].tokenizer);
    std::vector<std::string> tokens = tokenize_text(phrase, tok);
    if (tokens.empty()) return zero_all ? tq_all() : tq_none();
    return phrase_prefix_leaf(cx, (uint32_t)f, tokens, max_expansions);
  }
  if (type == "range") return range_query(cx, q.str_or("field", ""), q.get("lower_bound"), q.get("upper_bound"));
  if (type == "field_presence") {
    std::string field = q.str_or("field", "");
    int c = cx.img.find_column(field);
    if (c < 0) return tq_none();
    TQ t;
    t.kind = TQ::Exists;
    t.column = (uint32_t)c;
    return t;
  }
  if (type == "wildcard") {
    const std::string field = q.str_or("field", ""), value = q.str_or("value", "");
    const bool lenient = q.bool_or("lenient", false), ci = q.bool_or("case_insensitive", false);
    const int f = cx.img.find_field(field);
    if (is_ip_field(cx, field)) fail(QWGPU_EINVALID_QUERY, "invalid query: trying to run a Wildcard query on a non-text field");
    if (f < 0) {
      if (cx.img.find_column(field) >= 0 && cx.img.columns[cx.img.find_column(field)].type != QW_COL_STR)
        fail(QWGPU_EINVALID_QUERY, "invalid query: trying to run a Wildcard query on a non-text field");
      bool known = false;
      for (auto& fd : cx.dm.fields) if (fd.name == field) { known = true; if (fd.type != "text" && fd.type != "json") fail(QWGPU_EINVALID_QUERY, "invalid query: trying to run a Wildcard query on a non-text field"); }
      if (lenient || known) return tq_none();  // (declared in the doc mapping but without a single term in this split)
      fail(QWGPU_EINVALID_QUERY, "invalid query: field does not exist: `%s`", field.c_str());
    }
    refuse_const_score_under_ranking(cx, "wildcard");
    // sub_query_parts_to_regex: text parts go through the field tokenizer's NORMALIZER (raw: unchanged; default:
    // lower-cased), `*` = `.*`, `?` = `.`; case_insensitive = the regex flag (?i) (ASCII folding here)
    std::vector<GlobPart> parts = parse_wildcard(value);
    const bool lower = cx.img.fields[f].tokenizer != QW_TOK_RAW;
    auto fold = [](std::string& t) { for (char& c : t) if ((unsigned char)c < 0x80) c = (char)tolower((unsigned char)c); };
    for (GlobPart& p : parts) if (p.kind == 0 && (lower || ci)) fold(p.text);
    TQ b;
    b.kind = TQ::Bool;
    const QwImgField& F = cx.img.fields[f];
    const int group = cx.groups++;
    std::string folded;
    for (uint32_t t = F.first_term; t < F.first_term + F.num_terms; t++) {
      const QwImgTerm& T = cx.img.terms[t];
      const uint8_t* bytes = cx.img.term_bytes + T.bytes_off;
      if (ci) { folded.assign((const char*)bytes, T.bytes_len); fold(folded); bytes = (const uint8_t*)folded.data(); }
      if (!glob_match(parts, 0, bytes, T.bytes_len, 0)) continue;
      TQ leaf;
      leaf.kind = TQ::Term;
      leaf.term_ord = t;
      leaf.group = group;
      b.should.push_back(std::move(leaf));
    }
    if (b.should.empty()) return tq_none();
    TQ outer;  // constant-score membership test, like term_set below
    outer.kind = TQ::Bool;
    outer.filter.push_back(std::move(b));
    return outer;
  }
  if (type == "term_set") {
    refuse_const_score_under_ranking(cx, "term_set");
    TQ b;
    b.kind = TQ::Bool;
    if (const Json* tpf = q.get("terms_per_field"))
      for (auto& kv : tpf->obj) {
        const int group = cx.groups++;  // one set group per field
        for (auto& v : kv.second.arr) {
          b.should.push_back(full_text(cx, kv.first, lit_str(v), "raw", "bool", false, 0, true));
          b.should.back().group = group;
        }
      }
    if (b.should.empty()) return tq_none();
    // TermSetQuery is a constant-score set membership test: wrap as filter so it never scores
    TQ outer;
    outer.kind = TQ::Bool;
    outer.filter.push_back(std::move(b));
    return outer;
  }
  if (type == "boost") {
    const Json* u = q.get("underlying");
    if (!u) fail(QWGPU_EINVALID_QUERY, "invalid query: boost without underlying query");
    TQ inner = simplify(build(cx, *u, depth + 1));
    const Json* b = q.get("boost");
    apply_boost(inner, b && b->is_num() ? (float)b->as_f64() : 1.0f);
    inner.opaque = true;
    return inner;
  }
  if (type == "cache") {
    // CacheNode (cache_node.rs): a QW_NODE_CACHE over the inner query, opaque to simplify like a boost. A request ranked
    // by _score reads scores the cache does not keep: the inner query is compiled in its place.
    const Json* inner = q.get("inner");
    if (!inner) fail(QWGPU_EINVALID_QUERY, "invalid query: cache node without inner query");
    if (cx.scoring) return build(cx, *inner, depth + 1);
    TQ c;
    c.kind = TQ::Cache;
    c.opaque = true;
    c.must.push_back(simplify(build(cx, *inner, depth + 1)));
    return c;
  }
  if (type == "user_input")
    fail(QWGPU_EINVALID_QUERY, "invalid query: user_input queries must be parsed by the root before reaching a leaf");
  if (type == "regex") return regex_leaf(cx, q.str_or("field", ""), q.str_or("regex", ""));
  fail(QWGPU_EINVALID_QUERY, "invalid query: unknown query type `%s`", type.c_str());
}

// ---- flatten TQ -> QwPlanNode[] (children contiguous) ----------------------------------------------
static void emit(const TQ& t, uint32_t occur, const ImageView& img, std::vector<QwPlanNode>& out, size_t idx) {
  QwPlanNode& n = out[idx];
  memset(&n, 0, sizeof n);
  n.occur = occur;
  n.boost = t.boost;
  n.min_should_match = 0xFFFFFFFFu;
  n.term_ord = 0xFFFFFFFFu;
  n.column = 0xFFFFFFFFu;
  switch (t.kind) {
    case TQ::All: n.kind = QW_NODE_ALL; break;
    case TQ::None: n.kind = QW_NODE_NONE; break;
    case TQ::Exists: n.kind = QW_NODE_EXISTS; n.column = t.column; break;
    case TQ::Range: n.kind = QW_NODE_RANGE; n.column = t.column; n.lo = t.lo; n.hi = t.hi; break;
    case TQ::Term: {
      n.kind = QW_NODE_TERM;
      n.term_ord = t.term_ord;
      if (t.term_ord != 0xFFFFFFFFu) {
        const QwImgTerm& it = img.terms[t.term_ord];
        n.field_id = it.field_id;
        // Bm25Weight: idf * (1 + K1), then boost_by(boost) (SURVEY.md Appendix A.3)
        float w = bm25_idf(it.doc_freq, img.hdr->num_docs) * (1.0f + BM25_K1);
        n.bm25_weight = w * t.boost;
      }
      break;
    }
    case TQ::Phrase: {
      // PhraseWeight: Bm25Weight::for_terms = (sum of the terms' idf, duplicates included) * (1 + K1) * boost
      n.kind = QW_NODE_PHRASE;
      float idf_sum = 0.0f;
      for (uint32_t ord : t.phrase_terms) idf_sum += bm25_idf(img.terms[ord].doc_freq, img.hdr->num_docs);
      const uint32_t field_id = img.terms[t.phrase_terms[0]].field_id;
      n.field_id = field_id;
      n.bm25_weight = idf_sum * (1.0f + BM25_K1) * t.boost;
      const size_t first = out.size();  // (`n` dangles after the resize below)
      out[idx].first_child = (uint32_t)first;
      out[idx].num_children = (uint32_t)t.phrase_terms.size();
      out.resize(first + t.phrase_terms.size());
      for (size_t k = 0; k < t.phrase_terms.size(); k++) {
        QwPlanNode& c = out[first + k];
        memset(&c, 0, sizeof c);
        c.kind = QW_NODE_TERM; c.occur = QW_OCCUR_MUST; c.boost = 1.0f; c.min_should_match = 0xFFFFFFFFu;
        c.term_ord = t.phrase_terms[k]; c.field_id = field_id; c.column = 0xFFFFFFFFu;
        c.bm25_weight = bm25_idf(img.terms[c.term_ord].doc_freq, img.hdr->num_docs) * (1.0f + BM25_K1);
        c.lo = k;  // position offset inside the phrase
      }
      break;
    }
    case TQ::PhrasePrefix: {
      // never scored (refused in scoring clauses under _score ranking): children = exact terms, then expansions
      n.kind = QW_NODE_PHRASE_PREFIX;
      const uint32_t field_id = img.terms[t.phrase_terms[0]].field_id;
      const size_t k = t.phrase_terms.size(), e = t.prefix_terms.size();
      n.field_id = field_id;
      n.lo = k;
      const size_t first = out.size();  // (`n` dangles after the resize below)
      out[idx].first_child = (uint32_t)first;
      out[idx].num_children = (uint32_t)(k + e);
      out.resize(first + k + e);
      for (size_t i = 0; i < k + e; i++) {
        QwPlanNode& c = out[first + i];
        memset(&c, 0, sizeof c);
        c.kind = QW_NODE_TERM; c.occur = QW_OCCUR_MUST; c.boost = 1.0f; c.min_should_match = 0xFFFFFFFFu;
        c.term_ord = i < k ? t.phrase_terms[i] : t.prefix_terms[i - k]; c.field_id = field_id; c.column = 0xFFFFFFFFu;
        c.bm25_weight = bm25_idf(img.terms[c.term_ord].doc_freq, img.hdr->num_docs) * (1.0f + BM25_K1);
        c.lo = i < k ? i : k;  // position offset inside the phrase; every expansion sits in the last slot
      }
      break;
    }
    case TQ::TermSet: {
      // never scored (refused in scoring clauses under _score ranking): children = the terms, ascending
      n.kind = QW_NODE_TERM_SET;
      const uint32_t field_id = img.terms[t.prefix_terms[0]].field_id;
      n.field_id = field_id;
      const size_t first = out.size(), e = t.prefix_terms.size();  // (`n` dangles after the resize below)
      out[idx].first_child = (uint32_t)first;
      out[idx].num_children = (uint32_t)e;
      out.resize(first + e);
      for (size_t i = 0; i < e; i++) {
        QwPlanNode& c = out[first + i];
        memset(&c, 0, sizeof c);
        c.kind = QW_NODE_TERM; c.occur = QW_OCCUR_SHOULD; c.boost = 1.0f; c.min_should_match = 0xFFFFFFFFu;
        c.term_ord = t.prefix_terms[i]; c.field_id = field_id; c.column = 0xFFFFFFFFu;
        c.bm25_weight = bm25_idf(img.terms[c.term_ord].doc_freq, img.hdr->num_docs) * (1.0f + BM25_K1);
      }
      break;
    }
    case TQ::ColSet: {
      // never scored (refused in scoring clauses under _score ranking): children = one RANGE lo == hi per value, ascending
      n.kind = QW_NODE_COL_SET;
      n.column = t.column;
      const size_t first = out.size(), e = t.set_values.size();  // (`n` dangles after the resize below)
      out[idx].first_child = (uint32_t)first;
      out[idx].num_children = (uint32_t)e;
      out.resize(first + e);
      for (size_t i = 0; i < e; i++) {
        QwPlanNode& c = out[first + i];
        memset(&c, 0, sizeof c);
        c.kind = QW_NODE_RANGE; c.occur = QW_OCCUR_SHOULD; c.boost = 1.0f; c.min_should_match = 0xFFFFFFFFu;
        c.term_ord = 0xFFFFFFFFu; c.column = t.column; c.lo = c.hi = t.set_values[i];
      }
      break;
    }
    case TQ::Cache: {
      n.kind = QW_NODE_CACHE;
      const size_t first = out.size();  // (`n` dangles after the resize below)
      out[idx].first_child = (uint32_t)first;
      out[idx].num_children = 1;
      out.resize(first + 1);
      emit(t.must[0], QW_OCCUR_MUST, img, out, first);
      break;
    }
    case TQ::Bool: {
      n.kind = QW_NODE_BOOL;
      if (t.has_msm) n.min_should_match = (uint32_t)t.msm;
      size_t first = out.size();
      size_t cnt = t.must.size() + t.must_not.size() + t.should.size() + t.filter.size();
      out[idx].first_child = (uint32_t)first;
      out[idx].num_children = (uint32_t)cnt;
      out.resize(first + cnt);
      size_t k = first;
      // clause order of the reference's BooleanQuery: must, must_not, should, then filters
      // (tantivy_query_ast.rs:352-372)
      for (auto& c : t.must) emit(c, QW_OCCUR_MUST, img, out, k++);
      for (auto& c : t.must_not) emit(c, QW_OCCUR_MUST_NOT, img, out, k++);
      for (auto& c : t.should) emit(c, QW_OCCUR_SHOULD, img, out, k++);
      for (auto& c : t.filter) emit(c, QW_OCCUR_FILTER, img, out, k++);
      break;
    }
  }
}

// ---- set groups -> set nodes (DESIGN §4.8) -------------------------------------------------------------
// A set group is the leaves of one wildcard, of one one-token prefix, or of one term_set on one field: TERM leaves of
// one text / indexed `ip` field, or RANGE lo == hi leaves of one fast column. Each compiles to one plan leaf per value,
// as a should clause, unless the plan would then not fit the window program: then groups become set nodes, the largest
// first (ties in query order), until it fits.

// The instructions and TERM instructions the plan at nodes[i] lowers to (lower_node, engine.cu), with every CACHE node
// lowered as its child: the lowering every plan with cache nodes also goes through
static void program_size(const std::vector<QwPlanNode>& nodes, uint32_t i, uint64_t& terms, uint64_t& instrs) {
  const QwPlanNode& n = nodes[i];
  if (n.kind == QW_NODE_CACHE) return program_size(nodes, n.first_child, terms, instrs);
  if (n.kind == QW_NODE_TERM) terms++;
  instrs += n.kind == QW_NODE_BOOL ? 2 : 1;  // a bool: its BOOL_BEGIN / BOOL_END around the children
  if (n.kind == QW_NODE_BOOL)
    for (uint32_t c = 0; c < n.num_children; c++) program_size(nodes, n.first_child + c, terms, instrs);
}
// lower_plan's root rule: a root that is not a bool gets a bool around it
static bool plan_fits(const std::vector<QwPlanNode>& nodes, bool scoring) {
  uint32_t root = 0;
  while (nodes[root].kind == QW_NODE_CACHE) root = nodes[root].first_child;
  uint64_t terms = 0, instrs = nodes[root].kind == QW_NODE_BOOL ? 0 : 2;
  program_size(nodes, root, terms, instrs);
  return qw_program_fits(terms, instrs);
}

static void group_sizes(const TQ& t, std::map<int, size_t>& sizes) {
  if (t.group >= 0) sizes[t.group]++;
  for (auto* vec : {&t.must, &t.should, &t.must_not, &t.filter})
    for (const TQ& c : *vec) group_sizes(c, sizes);
}

// The set node of a group's leaves: their present values, sorted and deduplicated; none present: match-nothing
static TQ set_node(const std::vector<TQ>& leaves) {
  TQ s;
  for (const TQ& l : leaves) {
    if (l.kind == TQ::Term && l.term_ord != 0xFFFFFFFFu) { s.kind = TQ::TermSet; s.prefix_terms.push_back(l.term_ord); }
    if (l.kind == TQ::Range) { s.kind = TQ::ColSet; s.column = l.column; s.set_values.push_back(l.lo); }
  }
  std::sort(s.prefix_terms.begin(), s.prefix_terms.end());
  s.prefix_terms.erase(std::unique(s.prefix_terms.begin(), s.prefix_terms.end()), s.prefix_terms.end());
  std::sort(s.set_values.begin(), s.set_values.end());
  s.set_values.erase(std::unique(s.set_values.begin(), s.set_values.end()), s.set_values.end());
  const size_t e = s.prefix_terms.size() + s.set_values.size();
  if (e > QW_MAX_SET_TERMS)
    fail(QWGPU_EUNSUPPORTED, "term set with %zu values in split (the GPU path takes at most %d)", e, QW_MAX_SET_TERMS);
  return e ? s : tq_none();
}

// Replaces the leaves of group g, wherever a clause list holds them, by their set node
static void group_to_set_node(TQ& t, int g) {
  for (auto* vec : {&t.must, &t.should, &t.must_not, &t.filter}) {
    std::vector<TQ> leaves, kept;
    size_t at = 0;
    for (TQ& c : *vec) {
      if (c.group != g) { kept.push_back(std::move(c)); continue; }
      if (leaves.empty()) at = kept.size();
      leaves.push_back(std::move(c));
    }
    if (!leaves.empty()) kept.insert(kept.begin() + at, set_node(leaves));
    *vec = std::move(kept);
    for (TQ& c : *vec) group_to_set_node(c, g);
  }
}

// The plan nodes of `root`, with as many set groups turned into set nodes as the window program needs
static std::vector<QwPlanNode> emit_fitted(TQ root, const Ctx& cx) {
  std::vector<QwPlanNode> nodes(1);
  emit(root, QW_OCCUR_MUST, cx.img, nodes, 0);
  if (plan_fits(nodes, cx.scoring)) return nodes;
  std::map<int, size_t> sizes;
  group_sizes(root, sizes);
  std::vector<std::pair<int, size_t>> order(sizes.begin(), sizes.end());  // (query order)
  std::stable_sort(order.begin(), order.end(), [](const auto& a, const auto& b) { return a.second > b.second; });
  for (const auto& g : order) {
    // (the whole root may be the group's one leaf)
    TQ holder;
    holder.kind = TQ::Bool;
    holder.must.push_back(std::move(root));
    group_to_set_node(holder, g.first);
    root = simplify(std::move(holder.must[0]));
    nodes.assign(1, QwPlanNode{});
    emit(root, QW_OCCUR_MUST, cx.img, nodes, 0);
    if (plan_fits(nodes, cx.scoring)) break;
  }
  return nodes;  // (a plan that still does not fit is refused by lowering)
}

// ---- search_after conversion (collector.rs:214-372) ---------------------------------------------------
enum SortFieldType { SFT_U64, SFT_I64, SFT_F64, SFT_DATETIME, SFT_BOOL };
static bool convert_to_u64_ff_val(const pb::SortValue& sv, uint32_t kind, int sft, uint32_t order, uint64_t* out) {
  using SV = pb::SortValue;
  const bool desc = order == QW_ORDER_DESC, asc = !desc;
  if (kind == QW_SORT_DOCID) {
    if (sv.kind != SV::U64) fail(QWGPU_EINVALID_ARG, "Internal error: Got non-U64 sort value for DocId.");
    *out = sv.u;
    return true;
  }
  if (kind == QW_SORT_SCORE) {
    if (sv.kind != SV::F64) fail(QWGPU_EINVALID_ARG, "Internal error: Got non-F64 sort value for Score.");
    *out = f64_to_u64(sv.f);
    return true;
  }
  auto dt = [](int64_t nanos) { return i64_to_u64(nanos); };
  switch (sv.kind) {
    case SV::U64: {
      uint64_t v = sv.u;
      switch (sft) {
        case SFT_U64: *out = v; return true;
        case SFT_I64: if (desc && v > (uint64_t)INT64_MAX) return false; *out = i64_to_u64((int64_t)std::min<uint64_t>(v, INT64_MAX)); return true;
        case SFT_F64: *out = f64_to_u64((double)v); return true;
        case SFT_DATETIME: if (desc && v > (uint64_t)INT64_MAX) return false; *out = dt((int64_t)std::min<uint64_t>(v, INT64_MAX)); return true;
        case SFT_BOOL: if (v > 1 && desc) return false; *out = v >= 1 ? 1 : 0; return true;
      }
      break;
    }
    case SV::I64: {
      int64_t v = sv.i;
      switch (sft) {
        case SFT_I64: *out = i64_to_u64(v); return true;
        case SFT_U64: if (v < 0 && asc) return false; *out = v < 0 ? 0 : (uint64_t)v; return true;
        case SFT_F64: *out = f64_to_u64((double)v); return true;
        case SFT_DATETIME: *out = dt(v); return true;
        case SFT_BOOL: if ((v > 1 && desc) || (v < 0 && asc)) return false; *out = std::min<int64_t>(std::max<int64_t>(v, 0), 1) == 1; return true;
      }
      break;
    }
    case SV::F64: {
      double v = sv.f;
      switch (sft) {
        case SFT_F64: *out = f64_to_u64(v); return true;
        case SFT_U64:
          if ((v < 0.0 && asc) || (v > 18446744073709551615.0 && desc)) return false;
          *out = v <= 0 ? 0 : (v >= 18446744073709551615.0 ? ~0ull : (uint64_t)v);
          return true;
        case SFT_I64: case SFT_DATETIME: {
          if ((v < -9223372036854775808.0 && asc) || (v > 9223372036854775807.0 && desc)) return false;
          int64_t i = v != v ? 0 : (v <= -9223372036854775808.0 ? INT64_MIN : (v >= 9223372036854775807.0 ? INT64_MAX : (int64_t)v));
          *out = sft == SFT_DATETIME ? dt(i) : i64_to_u64(i);
          return true;
        }
        case SFT_BOOL:
          if ((v > 1.0 && desc) || (v < 0.0 && asc)) return false;
          *out = std::min(std::max(v, 0.0), 1.0) >= 0.5;
          return true;
      }
      break;
    }
    case SV::Bool: {
      uint64_t v = sv.b;
      switch (sft) {
        case SFT_BOOL: case SFT_U64: *out = v; return true;
        case SFT_F64: *out = f64_to_u64((double)v); return true;
        case SFT_I64: *out = i64_to_u64((int64_t)v); return true;
        case SFT_DATETIME: *out = dt((int64_t)v); return true;
      }
      break;
    }
    default: break;
  }
  return false;
}

CompiledPlan compile_plan(const ImageView& img, const std::string& split_id, const pb::SearchRequest& req_in,
                          const DocMapperInfo& dm, const pb::SplitIdAndFooterOffsets* split_meta, const Json* parsed_ast) {
  pb::SearchRequest req = req_in;
  // rewrite_request (leaf.rs:712-729)
  if (req.max_hits == 0 && req.start_offset == 0) req.sort_fields.clear();
  Ctx cx{img, dm};
  for (const pb::SortField& sf : req.sort_fields) if (sf.field_name == "_score") cx.scoring = true;
  Json local_ast;
  if (!parsed_ast) { local_ast = parse_json(req.query_ast, QWGPU_EINVALID_QUERY); parsed_ast = &local_ast; }
  TQ root = build(cx, *parsed_ast, 0);
  // [start_timestamp, end_timestamp) folded into the AST as a filter on the timestamp field
  // (remove_redundant_timestamp_range, leaf.rs:841-946); the clause is skipped when the split's own
  // time range already lies inside the bounds
  if ((req.start_timestamp || req.end_timestamp) && !dm.timestamp_field.empty()) {
    bool need_lo = req.start_timestamp.has_value(), need_hi = req.end_timestamp.has_value();
    if (split_meta) {
      if (need_lo && split_meta->timestamp_start && *req.start_timestamp <= *split_meta->timestamp_start) need_lo = false;
      if (need_hi && split_meta->timestamp_end && *req.end_timestamp >= *split_meta->timestamp_end + 1) need_hi = false;
    }
    if (need_lo || need_hi) {
      int c = img.find_column(dm.timestamp_field);
      TQ range = tq_none();
      if (c >= 0) {
        uint64_t lo = 0, hi = ~0ull;
        int64_t prec = precision_ns(dm, dm.timestamp_field);
        if (need_lo) lo = i64_to_u64(truncate_ns(*req.start_timestamp * 1000000000ll, prec));
        if (need_hi) { uint64_t m = i64_to_u64(truncate_ns(*req.end_timestamp * 1000000000ll, prec)); hi = m == 0 ? 0 : m - 1; if (m == 0) lo = 1; }
        if (lo <= hi) range = range_leaf((uint32_t)c, lo, hi);
      }
      TQ outer;
      outer.kind = TQ::Bool;
      outer.must.push_back(std::move(root));
      outer.filter.push_back(std::move(range));
      root = std::move(outer);
    }
  }
  root = simplify(std::move(root));

  CompiledPlan cp;
  const std::vector<QwPlanNode> nodes = emit_fitted(std::move(root), cx);

  QwPlanHeader h;
  memset(&h, 0, sizeof h);
  h.magic = QW_PLAN_MAGIC;
  h.version = 1;
  h.num_nodes = (uint32_t)nodes.size();
  uint64_t k = req.max_hits + req.start_offset;
  if (k > 0xFFFFFFFFull) fail(QWGPU_EINVALID_ARG, "max_hits + start_offset too large");
  h.max_hits = (uint32_t)k;
  // sort_by_from_request (collector.rs:994-1030)
  if (req.sort_fields.size() > 2) fail(QWGPU_EINVALID_ARG, "Sort by more than 2 fields is not supported yet.");
  int sft[2] = {SFT_U64, SFT_U64};
  for (size_t i = 0; i < 2; i++) {
    h.sort[i].kind = i == 0 ? (uint32_t)QW_SORT_DOCID : (uint32_t)QW_SORT_NONE;
    h.sort[i].order = QW_ORDER_DESC;
    h.sort[i].column = 0xFFFFFFFFu;
    if (i >= req.sort_fields.size()) continue;
    const pb::SortField& sf = req.sort_fields[i];
    h.sort[i].order = sf.sort_order == 0 ? QW_ORDER_ASC : QW_ORDER_DESC;
    if (sf.field_name == "_score") h.sort[i].kind = QW_SORT_SCORE;
    else if (sf.field_name == "_shard_doc" || sf.field_name == "_doc") h.sort[i].kind = QW_SORT_DOCID;
    else {
      h.sort[i].kind = QW_SORT_COLUMN;
      int c = img.find_column(sf.field_name);
      if (c >= 0) {
        uint32_t t = img.columns[c].type;
        if (t == QW_COL_STR) fail(QWGPU_EINVALID_ARG, "Unsupported sort field type `Str`.");
        if (t == QW_COL_IP) fail(QWGPU_EINVALID_ARG, "Unsupported sort field type `IpAddr`.");
        if (t == QW_COL_BYTES) fail(QWGPU_EUNSUPPORTED, "sorting on bytes field `%s` is not supported on the GPU path", sf.field_name.c_str());
        h.sort[i].column = (uint32_t)c;
        sft[i] = t == QW_COL_U64 ? SFT_U64 : t == QW_COL_I64 ? SFT_I64 : t == QW_COL_F64 ? SFT_F64 : t == QW_COL_BOOL ? SFT_BOOL : SFT_DATETIME;
      }
    }
  }
  h.scoring = (h.sort[0].kind == QW_SORT_SCORE || h.sort[1].kind == QW_SORT_SCORE) ? 1 : 0;
  // SearchAfterSegment::new (top_k_collector.rs:829-872)
  if (req.search_after) {
    const pb::PartialHit& sa = *req.search_after;
    QwSearchAfter& o = h.search_after;
    o.present = 1;
    bool disabled = false;
    if (sa.has_sv1 && sa.sv1.kind != pb::SortValue::None) {
      uint64_t v;
      if (convert_to_u64_ff_val(sa.sv1, h.sort[0].kind, sft[0], h.sort[0].order, &v)) { o.has_v1 = 1; o.v1 = v; }
      else disabled = true;  // out of bounds: search_after disabled, everything matches
    }
    if (!disabled && sa.has_sv2 && sa.sv2.kind != pb::SortValue::None) {
      if (h.sort[1].kind == QW_SORT_NONE) fail(QWGPU_EINVALID_ARG, "Internal error: Got sort_value2, but no sort extractor");
      uint64_t v;
      if (convert_to_u64_ff_val(sa.sv2, h.sort[1].kind, sft[1], h.sort[1].order, &v)) { o.has_v2 = 1; o.v2 = v; }
    }
    if (disabled) memset(&o, 0, sizeof o);
    else {
      o.compare_on_equal = !sa.split_id.empty();
      o.doc_id = sa.doc_id;
      if (o.compare_on_equal) {
        int c = split_id.compare(sa.split_id);
        c = c < 0 ? -1 : (c > 0 ? 1 : 0);
        if (c == 0) c = sa.segment_ord > 0 ? -1 : 0;  // our segment_ord is always 0
        o.precomp_order = h.sort[0].order == QW_ORDER_DESC ? c : -c;
      }
    }
  }
  // aggregations
  std::vector<QwAggNode> aggs;
  if (req.aggregation_request && !req.aggregation_request->empty()) {
    cp.agg_request = parse_agg_request(*req.aggregation_request);
    // Jaeger's trace search sends the find_trace_ids collector with max_hits 0; the GPU path runs it alone
    if (is_trace_ids_request(cp.agg_request) && h.max_hits > 0)
      fail(QWGPU_EUNSUPPORTED, "find_trace_ids combined with max_hits > 0 is not implemented on the GPU path");
    aggs = lower_aggs(cp.agg_request, img, cp.agg_bindings, &dm);
  }
  h.num_aggs = (uint32_t)aggs.size();
  h.count_only = (h.max_hits == 0 && aggs.empty()) ? 1 : 0;
  cp.bytes.assign((const char*)&h, sizeof h);
  cp.bytes.append((const char*)nodes.data(), nodes.size() * sizeof(QwPlanNode));
  if (!aggs.empty()) cp.bytes.append((const char*)aggs.data(), aggs.size() * sizeof(QwAggNode));
  cp.header = h;
  for (int i = 0; i < 2; i++) cp.sort_field_type[i] = sft[i];
  return cp;
}

}  // namespace qw
