// common.h — small shared helpers for the host side of libqwgpu (errors, value mappings, image view).
#pragma once
#include <cmath>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/qwgpu.h"
#include "device_types.h"

namespace qw {

// Error carrying a QWGPU_E* code; converted to return codes + thread-local message at the C ABI.
struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};
[[noreturn]] inline void fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  throw Error(code, buf);
}
void set_last_error(const std::string& msg);

// ---- raw-space boundary tables ---------------------------------------------------------------
// The smallest raw value in [lo, hi] for which `at_least` holds, a predicate monotone in the raw value (false, then
// true); hi itself is taken to hold and is never evaluated
template <class F>
inline uint64_t first_raw(uint64_t lo, uint64_t hi, F&& at_least) {
  while (lo < hi) {
    const uint64_t mid = lo + (hi - lo) / 2;
    if (at_least(mid)) hi = mid; else lo = mid + 1;
  }
  return lo;
}
// The boundary table of histogram node d over column c (DAgg::bounds, the fast aggregation paths): appends bounds[k]
// for k = 0..nb, the smallest raw value in [0, max_raw + 1] whose bucket, clamped to [-1, nb], is >= k. The bucket
// comes from qw_hist_pos as in agg_bucket, and is monotone in the raw value, so the device finds a raw value's bucket
// in the table without f64 arithmetic and lands where agg_bucket would. max_raw = the largest raw value present:
// searching beyond would leave the value domain (f64 columns: bit patterns past the maximum are NaNs and break the
// order).
inline void hist_bounds(const DCol& c, uint64_t max_raw, const DAgg& d, std::vector<uint64_t>& out) {
  const int64_t nb = d.num_buckets;
  auto bucket = [&](uint64_t raw) -> int64_t {
    const unsigned __int128 wide = (unsigned __int128)c.gcd * raw + c.min_value;  // saturate beyond the column's range
    const double val = qw_mapped_to_f64(c.type, wide > (unsigned __int128)~0ull ? ~0ull : (uint64_t)wide);
    if (d.has_bounds) {
      if (!(val >= d.bound_min)) return -1;
      if (!(val <= d.bound_max)) return nb;
    }
    const double pos = qw_hist_pos(val, d.offset, d.interval);
    if (!(pos >= -9.0e18)) return -1;
    if (!(pos <= 9.0e18)) return nb;
    const int64_t idx = (int64_t)pos - d.base_pos;
    return idx < 0 ? -1 : (idx >= nb ? nb : idx);
  };
  const uint64_t raw_end = max_raw == ~0ull ? max_raw : max_raw + 1;
  uint64_t lo = 0;
  for (int64_t k = 0; k <= nb; k++) {
    // (2^64 is not representable: an edge that no raw value reaches saturates at ~0)
    lo = max_raw == ~0ull && bucket(~0ull) < k ? ~0ull : first_raw(lo, raw_end, [&](uint64_t raw) { return bucket(raw) >= k; });
    out.push_back(lo);
  }
}

// ---- BM25 constants (tantivy Bm25Weight; SURVEY.md Appendix A.3) -------------------------------
constexpr float BM25_K1 = 1.2f;
constexpr float BM25_B = 0.75f;
inline float bm25_idf(uint64_t doc_freq, uint64_t doc_count) {
  float x = ((float)(doc_count - doc_freq) + 0.5f) / ((float)doc_freq + 0.5f);
  return logf(1.0f + x);
}

// ---- read-only view over a split image -------------------------------------------------------
struct ImageView {
  const uint8_t* base = nullptr;
  uint64_t len = 0;
  const QwImgHeader* hdr = nullptr;
  const QwImgField* fields = nullptr;
  const QwImgTerm* terms = nullptr;
  const QwImgColumn* columns = nullptr;
  const uint8_t* term_bytes = nullptr;
  const uint8_t* strings = nullptr;
  const uint8_t* data = nullptr;

  void open(const uint8_t* p, uint64_t n) {
    if (n < sizeof(QwImgHeader)) fail(QWGPU_EINVALID_ARG, "split image too small");
    const QwImgHeader* h = (const QwImgHeader*)p;
    if (h->magic != QW_IMG_MAGIC) fail(QWGPU_EINVALID_ARG, "bad split image magic");
    if (h->version != QW_IMG_VERSION) fail(QWGPU_EINVALID_ARG, "split image version %u (this library reads version %u)", h->version, QW_IMG_VERSION);
    if (h->total_len > n) fail(QWGPU_EINVALID_ARG, "split image truncated");
    // every section lies inside the image; every data-relative range inside the data region (those offsets
    // become device pointers in the kernels)
    const uint64_t tl = h->total_len;
    auto inside = [](uint64_t off, uint64_t count, uint64_t size, uint64_t limit) {
      return off <= limit && count <= (limit - off) / (size ? size : 1);
    };
    if (!inside(h->fields_off, h->num_fields, sizeof(QwImgField), tl) || !inside(h->terms_off, h->num_terms, sizeof(QwImgTerm), tl) ||
        !inside(h->columns_off, h->num_columns, sizeof(QwImgColumn), tl) || !inside(h->term_bytes_off, h->term_bytes_len, 1, tl) ||
        !inside(h->strings_off, h->strings_len, 1, tl) || !inside(h->data_off, h->data_len, 1, tl) || (h->data_len & 15))
      fail(QWGPU_EINVALID_ARG, "split image: a section lies outside the image");
    base = p;
    len = n;
    hdr = h;
    fields = (const QwImgField*)(p + h->fields_off);
    terms = (const QwImgTerm*)(p + h->terms_off);
    columns = (const QwImgColumn*)(p + h->columns_off);
    term_bytes = p + h->term_bytes_off;
    strings = p + h->strings_off;
    data = p + h->data_off;
    const uint64_t dl = h->data_len, nd = h->num_docs;
    for (uint32_t f = 0; f < h->num_fields; f++) {
      const QwImgField& F = fields[f];
      if (!inside(F.name_off, F.name_len, 1, h->strings_len) || !inside(F.first_term, F.num_terms, 1, h->num_terms) ||
          ((F.flags & QW_FIELD_HAS_FIELDNORMS) && !inside(F.fieldnorm_off, nd, 1, dl)))
        fail(QWGPU_EINVALID_ARG, "split image: field %u points outside the image", f);
    }
    for (uint32_t t = 0; t < h->num_terms; t++) {
      const QwImgTerm& T = terms[t];
      const uint64_t nwin = T.win_shift < 32 ? ((nd + (1ull << T.win_shift) - 1) >> T.win_shift) : 0;
      if (!inside(T.bytes_off, T.bytes_len, 1, h->term_bytes_len) || T.field_id >= h->num_fields ||
          T.num_blocks != (T.doc_freq + 127) / 128 || T.doc_freq > nd || !inside(T.skip_off, T.num_blocks, sizeof(QwSkip), dl) ||
          !inside(T.data_off, T.data_len, 1, dl) || !inside(T.widx_off, nwin, sizeof(QwWinIdx), dl) ||
          !inside(T.sub_off, T.num_blocks, sizeof(QwSubIdx), dl) || T.tf_len > T.data_len || T.fn_len > T.data_len ||
          (T.pidx_off && (!inside(T.pidx_off, (uint64_t)T.num_blocks + 1, 4, dl) || !inside(T.pos_off, 0, 4, dl))))
        fail(QWGPU_EINVALID_ARG, "split image: term %u points outside the image", t);
    }
    for (uint32_t c = 0; c < h->num_columns; c++) {
      const QwImgColumn& C = columns[c];
      if (!inside(C.name_off, C.name_len, 1, h->strings_len) || !inside(C.values_off, C.values_len, 1, dl) ||
          !inside(C.index_off, C.index_len, 1, dl) || !inside(C.dict_off, C.dict_len, 1, h->strings_len) || C.bits > 64 ||
          C.values_len < (C.num_vals * C.bits + 7) / 8)
        fail(QWGPU_EINVALID_ARG, "split image: column %u points outside the image", c);
    }
  }
  std::string field_name(uint32_t f) const {
    return std::string((const char*)strings + fields[f].name_off, fields[f].name_len);
  }
  std::string column_name(uint32_t c) const {
    return std::string((const char*)strings + columns[c].name_off, columns[c].name_len);
  }
  int find_field(const std::string& name) const {
    for (uint32_t f = 0; f < hdr->num_fields; f++)
      if (field_name(f) == name) return (int)f;
    return -1;
  }
  int find_column(const std::string& name) const {
    for (uint32_t c = 0; c < hdr->num_columns; c++)
      if (column_name(c) == name) return (int)c;
    return -1;
  }
  // binary search in the (field, bytes)-sorted dictionary; returns term ord or -1
  int find_term(uint32_t field, const uint8_t* bytes, uint32_t n) const {
    const QwImgField& f = fields[field];
    int lo = (int)f.first_term, hi = (int)(f.first_term + f.num_terms) - 1;
    while (lo <= hi) {
      int mid = (lo + hi) / 2;
      const QwImgTerm& t = terms[mid];
      uint32_t m = t.bytes_len < n ? t.bytes_len : n;
      int c = memcmp(term_bytes + t.bytes_off, bytes, m);
      if (c == 0) c = (t.bytes_len < n) ? -1 : (t.bytes_len > n ? 1 : 0);
      if (c == 0) return mid;
      if (c < 0) lo = mid + 1; else hi = mid - 1;
    }
    return -1;
  }
  // dictionary of a STR column
  void dict_term(const QwImgColumn& c, uint32_t ord, const uint8_t** p, uint32_t* n) const {
    const uint32_t* offs = (const uint32_t*)(strings + c.dict_off);
    const uint8_t* bytes = strings + c.dict_off + 4ull * (c.dict_num_terms + 1);
    *p = bytes + offs[ord];
    *n = offs[ord + 1] - offs[ord];
  }
  // ordinal of the first dictionary term >= key (lower bound); == dict_num_terms if none
  uint32_t dict_lower_bound(const QwImgColumn& c, const uint8_t* key, uint32_t n, bool* exact) const {
    uint32_t lo = 0, hi = c.dict_num_terms;
    *exact = false;
    while (lo < hi) {
      uint32_t mid = (lo + hi) / 2;
      const uint8_t* p; uint32_t m;
      dict_term(c, mid, &p, &m);
      uint32_t k = m < n ? m : n;
      int cmp = memcmp(p, key, k);
      if (cmp == 0) cmp = (m < n) ? -1 : (m > n ? 1 : 0);
      if (cmp < 0) lo = mid + 1; else { if (cmp == 0) *exact = true; hi = mid; }
    }
    return lo;
  }
};

// ---- aggregation cell layouts (aggs.cpp) ------------------------------------------------------
// The engine lays out a plan's cells and the host reads them back by the same rules.
// Dense (QwAggCell doc in qwgpu_format.h): total cells of the plan's aggregation nodes and each node's first cell;
// fails above QW_AGG_DENSE_MAX_CELLS.
uint64_t agg_cell_layout(const QwAggNode* aggs, uint32_t n, std::vector<uint32_t>* bases);
// Hashed (qw_agg_hashed): guaranteed upper bound on a split's distinct cells, the table slots and device bytes of a
// table of `cap` cells; agg_hashed_layout returns the bound and fails with QWGPU_EUNSUPPORTED when the table at the
// bound exceeds QWGPU_HASHED_MAX_BYTES
uint64_t agg_hashed_bound(const QwAggNode* aggs, uint32_t n, const ImageView& img);
uint32_t agg_hashed_slots(uint64_t cap);
uint64_t agg_hashed_table_bytes(uint64_t cap);
uint64_t agg_hashed_layout(const QwAggNode* aggs, uint32_t n, const ImageView& img, const char* split_id);

}  // namespace qw
