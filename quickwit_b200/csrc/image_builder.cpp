// image_builder.cpp — writer of the split image (include/qwgpu_format.h) + the synthetic
// hdfs-logs-shaped split generator used by bench.py and the full-size parity tests.
//
// The image is what `qwgpu_split_register` uploads to HBM. It plays the role of the tantivy
// segment files inside a Quickwit `.split` (SURVEY.md Appendix A.1/A.2/A.5); a real-split
// ingester (SURVEY.md §8f-2) would call this same writer after parsing `.idx/.fast/.fieldnorm`.
#include <algorithm>
#include <memory>
#include <numeric>

#include "common.h"

namespace qw {

// tantivy fieldnorm table == Lucene SmallFloat.byte4ToInt: ids below 24 are exact, above that a
// 3-bit-mantissa float (SURVEY.md Appendix A.3 "256-entry monotone table").
static uint32_t int4_to_long(uint32_t i) {
  uint32_t bits = i & 0x07, shift = (i >> 3);
  if (shift == 0) return bits;
  return (bits | 0x08) << (shift - 1);
}
uint32_t id_to_fieldnorm(uint8_t id) {
  const uint32_t kFree = 24;
  if (id < kFree) return id;
  return kFree + int4_to_long(id - kFree);
}
uint8_t fieldnorm_to_id(uint32_t fieldnorm) {
  // largest id with table[id] <= fieldnorm
  int lo = 0, hi = 255;
  while (lo < hi) {
    int mid = (lo + hi + 1) / 2;
    if (id_to_fieldnorm((uint8_t)mid) <= fieldnorm) lo = mid; else hi = mid - 1;
  }
  return (uint8_t)lo;
}

static inline uint32_t bits_needed(uint64_t v) { return v == 0 ? 0 : 64 - __builtin_clzll(v); }

// BitPacker4x-style interleaved packing of 128 values at `bits` bits => 16*bits bytes.
static void pack_block_4x(const uint32_t* v, uint32_t bits, uint8_t* out) {
  if (bits == 0) return;
  uint32_t* w = (uint32_t*)out;  // w[4*j + lane]
  memset(out, 0, 16 * bits);
  for (uint32_t i = 0; i < QW_BLOCK_LEN; i++) {
    uint32_t lane = i & 3, k = i >> 2;
    uint64_t bitpos = (uint64_t)k * bits;
    uint32_t wi = (uint32_t)(bitpos >> 5), sh = (uint32_t)(bitpos & 31);
    uint64_t val = (uint64_t)v[i] << sh;
    w[4 * wi + lane] |= (uint32_t)val;
    if (sh + bits > 32) w[4 * (wi + 1) + lane] |= (uint32_t)(val >> 32);
  }
}

struct BField {
  std::string name;
  uint32_t flags, tokenizer;
  uint64_t total_tokens;
  std::vector<uint8_t> fieldnorms;
};
struct BTerm {
  uint32_t field;
  std::string bytes;
  uint32_t doc_freq;
  uint32_t win_shift;
  uint64_t tf_len = 0, fn_len = 0;
  std::vector<QwSkip> skips;
  std::vector<QwSubIdx> subs;
  std::vector<uint32_t> first_docs;  // first doc of each block
  std::vector<uint8_t> data;
  std::vector<QwWinIdx> widx;
  std::vector<uint32_t> positions;  // fields with positions: tf[i] ascending token positions per posting
  std::vector<uint32_t> first_pos;  // [num_blocks + 1] index into `positions`
};
struct BColumn {
  std::string name;
  uint32_t type, card;
  uint64_t minv, maxv, gcd, num_vals;
  uint32_t bits, dict_n;
  std::vector<uint8_t> values;  // packed
  std::vector<uint8_t> index;
  std::vector<uint8_t> dict;  // offs[n+1] + bytes
};

}  // namespace qw

struct qwgpu_imgb {
  uint32_t num_docs;
  std::vector<qw::BField> fields;
  std::vector<qw::BTerm> terms;
  std::vector<qw::BColumn> columns;
};

namespace qw {

static void add_term(qwgpu_imgb* b, uint32_t field_id, const uint8_t* term, uint32_t term_len,
                     const uint32_t* docs, const uint32_t* tfs, uint32_t n, const uint32_t* positions = nullptr, uint64_t n_positions = 0) {
  if (field_id >= b->fields.size()) fail(QWGPU_EINVALID_ARG, "add_term: bad field id");
  if (n == 0) return;
  if (b->fields[field_id].tokenizer == QW_TOK_IP && term_len != 16) fail(QWGPU_EINVALID_ARG, "add_term: an ip field's terms are 16-byte addresses");
  bool has_freqs = (b->fields[field_id].flags & QW_FIELD_HAS_FREQS) != 0;
  const bool has_pos = (b->fields[field_id].flags & QW_FIELD_HAS_POSITIONS) != 0;
  if (has_pos) {
    if (!has_freqs || !tfs || !positions) fail(QWGPU_EINVALID_ARG, "add_term: a field with positions needs tfs and positions");
    uint64_t total = 0;
    for (uint32_t i = 0; i < n; i++) {
      if (tfs[i] == 0) fail(QWGPU_EINVALID_ARG, "add_term: tf 0");
      for (uint32_t k = 1; k < tfs[i]; k++)
        if (total + k >= n_positions || positions[total + k] <= positions[total + k - 1]) fail(QWGPU_EINVALID_ARG, "add_term: positions of a posting must be strictly increasing");
      total += tfs[i];
    }
    if (total != n_positions) fail(QWGPU_EINVALID_ARG, "add_term: %llu positions for a tf sum of %llu", (unsigned long long)n_positions, (unsigned long long)total);
  }
  bool has_fn = (b->fields[field_id].flags & QW_FIELD_HAS_FIELDNORMS) != 0;
  const std::vector<uint8_t>& fnorms = b->fields[field_id].fieldnorms;
  BTerm t;
  t.field = field_id;
  t.bytes.assign((const char*)term, term_len);
  t.doc_freq = n;
  uint32_t nblocks = (n + QW_BLOCK_LEN - 1) / QW_BLOCK_LEN;
  t.skips.resize(nblocks);
  uint32_t prev = QW_NO_PREV_DOC;
  uint32_t deltas[QW_BLOCK_LEN], tfv[QW_BLOCK_LEN];
  for (uint32_t blk = 0; blk < nblocks; blk++) {
    uint32_t start = blk * QW_BLOCK_LEN, cnt = std::min(QW_BLOCK_LEN, n - start);
    uint32_t maxd = 0, maxtf = 0, p = prev;
    for (uint32_t i = 0; i < QW_BLOCK_LEN; i++) {
      if (i < cnt) {
        uint32_t d = docs[start + i];
        if (!(p == QW_NO_PREV_DOC || d > p)) fail(QWGPU_EINVALID_ARG, "add_term: docs not strictly increasing");
        if (d >= b->num_docs) fail(QWGPU_EINVALID_ARG, "add_term: doc id out of range");
        deltas[i] = d - p - 1;  // mod 2^32
        p = d;
        tfv[i] = has_freqs ? (tfs ? tfs[start + i] : 1u) : 0u;
        maxd = std::max(maxd, deltas[i]);
        maxtf = std::max(maxtf, tfv[i]);
      } else {
        deltas[i] = 0;
        tfv[i] = 0;
      }
    }
    QwSkip& s = t.skips[blk];
    s.last_doc = docs[start + cnt - 1];
    s.prev_last_doc = prev;
    s.byte_off = (uint32_t)t.data.size();
    s.doc_bits = (uint8_t)bits_needed(maxd);
    s.tf_bits = has_freqs ? (uint8_t)bits_needed(maxtf) : 0;
    s.count = (uint16_t)cnt;
    size_t off = t.data.size();
    t.data.resize(off + 16u + 16u * (s.doc_bits + s.tf_bits) + (has_fn ? QW_BLOCK_LEN : 0u));
    memcpy(t.data.data() + off, &s, 16);  // inline header
    pack_block_4x(deltas, s.doc_bits, t.data.data() + off + 16u);
    pack_block_4x(tfv, s.tf_bits, t.data.data() + off + 16u + 16u * s.doc_bits);
    if (has_fn) {
      // per-posting fieldnorm ids (zero padded): one contiguous byte stream per block for BM25
      uint8_t* fb = t.data.data() + off + 16u + 16u * (s.doc_bits + s.tf_bits);
      for (uint32_t i = 0; i < cnt; i++) fb[i] = fnorms[docs[start + i]];
      t.fn_len += QW_BLOCK_LEN;
    }
    {
      QwSubIdx si;
      for (uint32_t k = 1; k <= 3; k++) si.ck[k - 1] = docs[start + std::min(32u * k, cnt) - 1] - prev;  // mod 2^32
      si.span = s.last_doc - prev;
      t.subs.push_back(si);
    }
    t.first_docs.push_back(docs[start]);
    t.tf_len += 16u * s.tf_bits;
    prev = s.last_doc;
  }
  if (has_pos) {
    t.positions.assign(positions, positions + n_positions);
    uint32_t acc = 0;
    for (uint32_t blk = 0; blk < nblocks; blk++) {
      t.first_pos.push_back(acc);
      for (uint32_t i = blk * QW_BLOCK_LEN; i < std::min(n, (blk + 1) * QW_BLOCK_LEN); i++) acc += tfs[i];
    }
    t.first_pos.push_back(acc);
  }
  // window index: granularity 2^win_shift docs, about <= 2 entries per block, never below 4096 docs
  uint32_t shift = QW_MIN_WIN_SHIFT;
  while ((((uint64_t)b->num_docs + (1ull << shift) - 1) >> shift) > 2ull * nblocks && shift < 31) shift++;
  t.win_shift = shift;
  uint32_t nwin = (uint32_t)(((uint64_t)b->num_docs + (1ull << shift) - 1) >> shift);
  t.widx.resize(nwin);
  uint32_t lo = 0;  // first block with last_doc >= window start
  for (uint32_t j = 0; j < nwin; j++) {
    uint64_t wstart = (uint64_t)j << shift, wend = wstart + (1ull << shift);
    while (lo < nblocks && t.skips[lo].last_doc < wstart) lo++;
    uint32_t hi = lo;  // one past the last block with first_doc < window end
    while (hi < nblocks && t.first_docs[hi] < wend) hi++;
    uint32_t sb = lo < nblocks ? t.skips[lo].byte_off : (uint32_t)t.data.size();
    uint32_t eb = hi < nblocks ? t.skips[hi].byte_off : (uint32_t)t.data.size();
    if (hi <= lo) eb = sb;
    t.widx[j].start = sb;
    t.widx[j].end = eb;
    t.widx[j].first_block = lo;
    t.widx[j].end_block = hi > lo ? hi : lo;
  }
  b->terms.push_back(std::move(t));
}

static uint64_t gcd64(uint64_t a, uint64_t b) {
  while (b) { uint64_t t = a % b; a = b; b = t; }
  return a;
}

static void add_column(qwgpu_imgb* b, const char* name, uint32_t type, uint32_t card,
                       const uint64_t* values, uint64_t num_vals, const uint32_t* index,
                       const uint8_t* dict_bytes, const uint32_t* dict_offs, uint32_t dict_n) {
  BColumn c;
  c.name = name;
  c.type = type;
  c.card = card;
  c.num_vals = num_vals;
  c.dict_n = dict_n;
  uint32_t nd = b->num_docs;
  if (card == QW_CARD_FULL && num_vals != nd) fail(QWGPU_EINVALID_ARG, "FULL column needs num_docs values");
  uint64_t mn = ~0ull, mx = 0;
  for (uint64_t i = 0; i < num_vals; i++) { mn = std::min(mn, values[i]); mx = std::max(mx, values[i]); }
  if (num_vals == 0) { mn = 0; mx = 0; }
  uint64_t g = 0;
  for (uint64_t i = 0; i < num_vals && g != 1; i++) g = gcd64(g, values[i] - mn);
  if (g == 0) g = 1;
  c.minv = mn; c.maxv = mx; c.gcd = g;
  c.bits = bits_needed((mx - mn) / g);
  uint64_t nbytes = (num_vals * c.bits + 7) / 8;
  c.values.assign(nbytes + 16, 0);
  if (c.bits) {
    uint64_t bitpos = 0;
    for (uint64_t i = 0; i < num_vals; i++, bitpos += c.bits) {
      uint64_t raw = (values[i] - mn) / g;
      uint64_t byte = bitpos >> 3; uint32_t sh = bitpos & 7;
      // write up to 9 bytes
      unsigned __int128 val = (unsigned __int128)raw << sh;
      for (uint32_t k = 0; k < 9 && (val >> (8 * k)) != 0; k++) c.values[byte + k] |= (uint8_t)(val >> (8 * k));
    }
  }
  if (card == QW_CARD_OPTIONAL) {
    uint32_t nw = (nd + 63) / 64;
    c.index.assign(8ull * nw + 4ull * (nw + 1), 0);
    uint64_t* present = (uint64_t*)c.index.data();
    uint32_t* rank = (uint32_t*)(c.index.data() + 8ull * nw);
    uint32_t prev = 0;
    for (uint64_t i = 0; i < num_vals; i++) {
      uint32_t d = index[i];
      if (d >= nd || (i > 0 && d <= prev)) fail(QWGPU_EINVALID_ARG, "OPTIONAL column: doc ids must be strictly increasing");
      present[d >> 6] |= 1ull << (d & 63);
      prev = d;
    }
    uint32_t acc = 0;
    for (uint32_t w = 0; w < nw; w++) { rank[w] = acc; acc += (uint32_t)__builtin_popcountll(present[w]); }
    rank[nw] = acc;
  } else if (card == QW_CARD_MULTI) {
    c.index.assign(4ull * (nd + 1), 0);
    memcpy(c.index.data(), index, 4ull * (nd + 1));
    if (((const uint32_t*)c.index.data())[nd] != num_vals) fail(QWGPU_EINVALID_ARG, "MULTI column: start[num_docs] != num_vals");
  }
  if (type == QW_COL_IP) {
    // ordinals into strictly increasing 16-byte addresses: byte order is address order
    for (uint32_t k = 0; k < dict_n; k++)
      if (dict_offs[k + 1] - dict_offs[k] != 16 || (k > 0 && memcmp(dict_bytes + dict_offs[k - 1], dict_bytes + dict_offs[k], 16) >= 0))
        fail(QWGPU_EINVALID_ARG, "ip column '%s': the dictionary must hold strictly increasing 16-byte addresses", name);
    if (num_vals && mx >= dict_n) fail(QWGPU_EINVALID_ARG, "ip column '%s': ordinal %llu outside a dictionary of %u addresses", name, (unsigned long long)mx, dict_n);
  }
  if (type == QW_COL_STR || type == QW_COL_BYTES || type == QW_COL_IP) {
    uint64_t blen = dict_n ? dict_offs[dict_n] : 0;
    c.dict.resize(4ull * (dict_n + 1) + blen);
    if (dict_n) memcpy(c.dict.data(), dict_offs, 4ull * (dict_n + 1));
    else memset(c.dict.data(), 0, 4);
    if (blen) memcpy(c.dict.data() + 4ull * (dict_n + 1), dict_bytes, blen);
  }
  b->columns.push_back(std::move(c));
}

static inline uint64_t align16(uint64_t x) { return (x + 15) & ~15ull; }

static void finish(qwgpu_imgb* b, uint8_t** out, uint64_t* out_len) {
  // sort terms by (field, bytes)
  std::vector<uint32_t> order(b->terms.size());
  std::iota(order.begin(), order.end(), 0);
  std::sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) {
    const BTerm &a = b->terms[x], &c = b->terms[y];
    if (a.field != c.field) return a.field < c.field;
    return a.bytes < c.bytes;
  });
  for (size_t i = 1; i < order.size(); i++) {
    const BTerm &a = b->terms[order[i - 1]], &c = b->terms[order[i]];
    if (a.field == c.field && a.bytes == c.bytes) fail(QWGPU_EINVALID_ARG, "duplicate term '%s'", a.bytes.c_str());
  }
  uint32_t nf = (uint32_t)b->fields.size(), nt = (uint32_t)b->terms.size(), nc = (uint32_t)b->columns.size();
  // strings blob
  std::vector<uint8_t> strings;
  auto put_str = [&](const std::string& s, uint32_t* off, uint32_t* len) {
    *off = (uint32_t)strings.size(); *len = (uint32_t)s.size();
    strings.insert(strings.end(), s.begin(), s.end());
  };
  std::vector<QwImgField> F(nf);
  std::vector<QwImgTerm> T(nt);
  std::vector<QwImgColumn> C(nc);
  memset(F.data(), 0, nf * sizeof(QwImgField));
  memset(T.data(), 0, nt * sizeof(QwImgTerm));
  memset(C.data(), 0, nc * sizeof(QwImgColumn));
  for (uint32_t f = 0; f < nf; f++) {
    put_str(b->fields[f].name, &F[f].name_off, &F[f].name_len);
    F[f].flags = b->fields[f].flags;
    F[f].tokenizer = b->fields[f].tokenizer;
    F[f].total_num_tokens = b->fields[f].total_tokens;
  }
  for (uint32_t c = 0; c < nc; c++) put_str(b->columns[c].name, &C[c].name_off, &C[c].name_len);
  for (uint32_t c = 0; c < nc; c++) {
    while (strings.size() & 3) strings.push_back(0);
    C[c].dict_off = strings.size();
    C[c].dict_len = b->columns[c].dict.size();
    strings.insert(strings.end(), b->columns[c].dict.begin(), b->columns[c].dict.end());
  }
  // term bytes
  std::vector<uint8_t> tbytes;
  // data region layout
  uint64_t doff = 0;
  for (uint32_t f = 0; f < nf; f++) {
    if (b->fields[f].flags & QW_FIELD_HAS_FIELDNORMS) { F[f].fieldnorm_off = doff; doff = align16(doff + b->num_docs + 16); }
  }
  for (uint32_t i = 0; i < nt; i++) {
    const BTerm& t = b->terms[order[i]];
    QwImgTerm& o = T[i];
    o.field_id = t.field;
    o.bytes_off = (uint32_t)tbytes.size();
    o.bytes_len = (uint32_t)t.bytes.size();
    tbytes.insert(tbytes.end(), t.bytes.begin(), t.bytes.end());
    o.doc_freq = t.doc_freq;
    o.num_blocks = (uint32_t)t.skips.size();
    o.skip_off = doff; doff = align16(doff + t.skips.size() * sizeof(QwSkip));
    o.data_off = doff; o.data_len = t.data.size(); doff = align16(doff + t.data.size() + 16);
    o.win_shift = t.win_shift;
    o.tf_len = t.tf_len;
    o.fn_len = t.fn_len;
    o.widx_off = doff; doff = align16(doff + t.widx.size() * sizeof(QwWinIdx));
    o.sub_off = doff; doff = align16(doff + t.subs.size() * sizeof(QwSubIdx));
    if (!t.first_pos.empty()) {
      o.pidx_off = doff; doff = align16(doff + t.first_pos.size() * 4);
      o.pos_off = doff; doff = align16(doff + t.positions.size() * 4 + 16);
    }
  }
  for (uint32_t f = 0; f < nf; f++) { F[f].first_term = 0; F[f].num_terms = 0; }
  for (uint32_t i = 0; i < nt; i++) {
    uint32_t f = T[i].field_id;
    if (F[f].num_terms == 0) F[f].first_term = i;
    F[f].num_terms++;
  }
  for (uint32_t c = 0; c < nc; c++) {
    const BColumn& bc = b->columns[c];
    QwImgColumn& o = C[c];
    o.type = bc.type; o.cardinality = bc.card;
    o.min_value = bc.minv; o.max_value = bc.maxv; o.gcd = bc.gcd; o.num_vals = bc.num_vals;
    o.bits = bc.bits; o.dict_num_terms = bc.dict_n;
    o.values_off = doff; o.values_len = bc.values.size(); doff = align16(doff + bc.values.size());
    o.index_off = doff; o.index_len = bc.index.size(); doff = align16(doff + bc.index.size());
  }
  uint64_t data_len = align16(doff);
  // file layout
  uint64_t off = sizeof(QwImgHeader);
  QwImgHeader H;
  memset(&H, 0, sizeof H);
  H.magic = QW_IMG_MAGIC; H.version = QW_IMG_VERSION; H.num_docs = b->num_docs;
  H.num_fields = nf; H.num_terms = nt; H.num_columns = nc;
  H.fields_off = off; off = align16(off + nf * sizeof(QwImgField));
  H.terms_off = off; off = align16(off + nt * sizeof(QwImgTerm));
  H.term_bytes_off = off; H.term_bytes_len = tbytes.size(); off = align16(off + tbytes.size());
  H.columns_off = off; off = align16(off + nc * sizeof(QwImgColumn));
  H.strings_off = off; H.strings_len = strings.size(); off = align16(off + strings.size());
  off = (off + 255) & ~255ull;
  H.data_off = off; H.data_len = data_len; off += data_len;
  H.total_len = off;
  uint8_t* img = (uint8_t*)calloc(1, off);
  if (!img) fail(QWGPU_EINTERNAL, "out of memory building split image (%llu bytes)", (unsigned long long)off);
  memcpy(img, &H, sizeof H);
  if (nf) memcpy(img + H.fields_off, F.data(), nf * sizeof(QwImgField));
  if (nt) memcpy(img + H.terms_off, T.data(), nt * sizeof(QwImgTerm));
  if (!tbytes.empty()) memcpy(img + H.term_bytes_off, tbytes.data(), tbytes.size());
  if (nc) memcpy(img + H.columns_off, C.data(), nc * sizeof(QwImgColumn));
  if (!strings.empty()) memcpy(img + H.strings_off, strings.data(), strings.size());
  uint8_t* data = img + H.data_off;
  for (uint32_t f = 0; f < nf; f++)
    if (b->fields[f].flags & QW_FIELD_HAS_FIELDNORMS) memcpy(data + F[f].fieldnorm_off, b->fields[f].fieldnorms.data(), b->num_docs);
  for (uint32_t i = 0; i < nt; i++) {
    const BTerm& t = b->terms[order[i]];
    memcpy(data + T[i].skip_off, t.skips.data(), t.skips.size() * sizeof(QwSkip));
    if (!t.data.empty()) memcpy(data + T[i].data_off, t.data.data(), t.data.size());
    if (!t.widx.empty()) memcpy(data + T[i].widx_off, t.widx.data(), t.widx.size() * sizeof(QwWinIdx));
    if (!t.subs.empty()) memcpy(data + T[i].sub_off, t.subs.data(), t.subs.size() * sizeof(QwSubIdx));
    if (!t.first_pos.empty()) {
      memcpy(data + T[i].pidx_off, t.first_pos.data(), t.first_pos.size() * 4);
      if (!t.positions.empty()) memcpy(data + T[i].pos_off, t.positions.data(), t.positions.size() * 4);
    }
  }
  for (uint32_t c = 0; c < nc; c++) {
    const BColumn& bc = b->columns[c];
    if (!bc.values.empty()) memcpy(data + C[c].values_off, bc.values.data(), bc.values.size());
    if (!bc.index.empty()) memcpy(data + C[c].index_off, bc.index.data(), bc.index.size());
  }
  *out = img;
  *out_len = off;
}

// ---- synthetic corpus --------------------------------------------------------------------------
// splitmix64 / xoshiro-free: a counter-based generator keeps every (split, stream) reproducible.
struct Rng {
  uint64_t s;
  explicit Rng(uint64_t seed) : s(seed) {}
  uint64_t next() {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
  }
  double uniform() { return (double)(next() >> 11) * (1.0 / 9007199254740992.0); }
};

static void synth_split(const qwgpu_synth_spec* sp, uint8_t** img, uint64_t* img_len) {
  uint32_t nd = sp->num_docs;
  std::unique_ptr<qwgpu_imgb> b(new qwgpu_imgb());
  b->num_docs = nd;
  uint64_t base_seed = sp->seed * 0x100000001B3ull + sp->split_ord * 0x9E3779B97F4A7C15ull;
  // body field: length 8..26 tokens (8-24 words + 1-2 unique block-id tokens; SURVEY.md §8d)
  {
    BField f;
    f.name = "body";
    f.flags = QW_FIELD_HAS_FREQS | QW_FIELD_HAS_FIELDNORMS;
    f.tokenizer = QW_TOK_DEFAULT;
    f.fieldnorms.resize(nd);
    Rng r(base_seed ^ 0xB0D1);
    uint64_t total = 0;
    for (uint32_t d = 0; d < nd; d++) {
      uint32_t len = 9 + (uint32_t)(r.next() % 18);
      total += len;
      f.fieldnorms[d] = fieldnorm_to_id(len);
    }
    f.total_tokens = total;
    b->fields.push_back(std::move(f));
  }
  // severity_text: raw tokenizer, no freqs/fieldnorms (record basic), also a fast STR column
  static const char* kSev[4] = {"DEBUG", "ERROR", "INFO", "WARN"};  // sorted = ordinals
  std::vector<uint64_t> sev(nd);
  {
    BField f;
    f.name = "severity_text";
    f.flags = 0;
    f.tokenizer = QW_TOK_RAW;
    f.total_tokens = nd;
    b->fields.push_back(std::move(f));
    Rng r(base_seed ^ 0x5E7);
    std::vector<uint32_t> docs[4];
    for (uint32_t d = 0; d < nd; d++) {
      double u = r.uniform();
      uint32_t o = u < 0.90 ? 2 : (u < 0.97 ? 3 : (u < 0.999 ? 1 : 0));  // INFO 90, WARN 7, ERROR 2.9, DEBUG 0.1
      sev[d] = o;
      docs[o].push_back(d);
    }
    for (int o = 0; o < 4; o++)
      add_term(b.get(), 1, (const uint8_t*)kSev[o], (uint32_t)strlen(kSev[o]), docs[o].data(), nullptr, (uint32_t)docs[o].size());
    std::string bytes; std::vector<uint32_t> offs{0};
    for (int o = 0; o < 4; o++) { bytes += kSev[o]; offs.push_back((uint32_t)bytes.size()); }
    add_column(b.get(), "severity_text", QW_COL_STR, QW_CARD_FULL, sev.data(), nd, nullptr, (const uint8_t*)bytes.data(), offs.data(), 4);
  }
  // body terms t0..t{n-1}: geometric gaps with P(doc has term) = frac; tf = 1 + geometric(0.35)
  for (uint32_t t = 0; t < sp->num_terms; t++) {
    double p = sp->term_fracs[t];
    if (p <= 0) continue;
    Rng r(base_seed ^ (0x7E4300ull + t));
    std::vector<uint32_t> docs, tfs;
    docs.reserve((size_t)(nd * p * 1.1) + 16);
    double inv = 1.0 / log1p(-std::min(p, 0.999999));
    int64_t d = -1;
    for (;;) {
      double u = r.uniform();
      int64_t gap = (p >= 1.0) ? 0 : (int64_t)floor(log1p(-u) * inv);
      d += 1 + gap;
      if (d >= (int64_t)nd) break;
      docs.push_back((uint32_t)d);
      uint32_t tf = 1;
      uint64_t x = r.next();
      while ((x & 0xFF) < 90 && tf < 12) { tf++; x >>= 8; }  // P(continue) ≈ 0.35
      tfs.push_back(tf);
    }
    char name[32];
    int n = snprintf(name, sizeof name, "t%u", t);
    add_term(b.get(), 0, (const uint8_t*)name, (uint32_t)n, docs.data(), tfs.data(), (uint32_t)docs.size());
  }
  // msg: optional text field with positions (phrase queries): 4..8 tokens per doc, Zipf(1) over "w<k>"
  if (sp->msg_vocab) {
    const uint32_t nv = sp->msg_vocab;
    const uint32_t fid = (uint32_t)b->fields.size();
    BField f;
    f.name = "msg";
    f.flags = QW_FIELD_HAS_FREQS | QW_FIELD_HAS_FIELDNORMS | QW_FIELD_HAS_POSITIONS;
    f.tokenizer = QW_TOK_DEFAULT;
    f.fieldnorms.resize(nd);
    std::vector<double> cdf(nv);
    double z = 0;
    for (uint32_t i = 0; i < nv; i++) { z += 1.0 / (double)(i + 1); cdf[i] = z; }
    struct Acc { std::vector<uint32_t> docs, tfs, pos; };
    std::vector<Acc> acc(nv);
    Rng r(base_seed ^ 0x3596);
    uint64_t total = 0;
    for (uint32_t d = 0; d < nd; d++) {
      const uint32_t len = 4 + (uint32_t)(r.next() % 5);
      total += len;
      f.fieldnorms[d] = fieldnorm_to_id(len);
      for (uint32_t t = 0; t < len; t++) {
        const double u = r.uniform() * z;
        uint32_t k = (uint32_t)(std::lower_bound(cdf.begin(), cdf.end(), u) - cdf.begin());
        if (k >= nv) k = nv - 1;
        Acc& a = acc[k];
        if (a.docs.empty() || a.docs.back() != d) { a.docs.push_back(d); a.tfs.push_back(0); }
        a.tfs.back()++;
        a.pos.push_back(t);
      }
    }
    f.total_tokens = total;
    b->fields.push_back(std::move(f));
    for (uint32_t k = 0; k < nv; k++) {
      char name[32];
      const int n = snprintf(name, sizeof name, "w%u", k);
      const Acc& a = acc[k];
      if (!a.docs.empty())
        add_term(b.get(), fid, (const uint8_t*)name, (uint32_t)n, a.docs.data(), a.tfs.data(), (uint32_t)a.docs.size(), a.pos.data(), a.pos.size());
    }
  }
  // timestamp: datetime, seconds precision, monotone within the split
  {
    std::vector<uint64_t> ts(nd);
    Rng r(base_seed ^ 0x715);
    // sorted uniform offsets via exponential spacings
    std::vector<double> acc(nd);
    double s = 0;
    for (uint32_t d = 0; d < nd; d++) { s += -log(1.0 - r.uniform()); acc[d] = s; }
    s += -log(1.0 - r.uniform());
    for (uint32_t d = 0; d < nd; d++) {
      int64_t secs = sp->ts_start_secs + (int64_t)(acc[d] / s * sp->ts_span_secs);
      ts[d] = i64_to_u64(secs * 1000000000ll);
    }
    add_column(b.get(), "timestamp", QW_COL_DATETIME, QW_CARD_FULL, ts.data(), nd, nullptr, nullptr, nullptr, 0);
  }
  // tenant_id: u64, Zipf(1.1) over num_tenants ids
  {
    uint32_t nt = sp->num_tenants ? sp->num_tenants : 100;
    std::vector<double> cdf(nt);
    double z = 0;
    for (uint32_t i = 0; i < nt; i++) { z += 1.0 / pow((double)(i + 1), 1.1); cdf[i] = z; }
    std::vector<uint64_t> tv(nd);
    Rng r(base_seed ^ 0x7E9A97);
    for (uint32_t d = 0; d < nd; d++) {
      double u = r.uniform() * z;
      uint32_t k = (uint32_t)(std::lower_bound(cdf.begin(), cdf.end(), u) - cdf.begin());
      if (k >= nt) k = nt - 1;
      tv[d] = 1000 + k;
    }
    add_column(b.get(), "tenant_id", QW_COL_U64, QW_CARD_FULL, tv.data(), nd, nullptr, nullptr, nullptr, 0);
  }
  finish(b.get(), img, img_len);
}

}  // namespace qw

// ---- C ABI ------------------------------------------------------------------------------------
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

extern "C" {

qwgpu_imgb* qwgpu_imgb_new(uint32_t num_docs) {
  qwgpu_imgb* b = new qwgpu_imgb();
  b->num_docs = num_docs;
  return b;
}
void qwgpu_imgb_free(qwgpu_imgb* b) { delete b; }

int qwgpu_imgb_add_field(qwgpu_imgb* b, const char* name, uint32_t flags, uint32_t tokenizer,
                         const uint8_t* fieldnorm_ids, uint64_t total_num_tokens) {
  QW_API_BEGIN
  qw::BField f;
  f.name = name;
  f.flags = flags;
  f.tokenizer = tokenizer;
  f.total_tokens = total_num_tokens;
  if (tokenizer == QW_TOK_IP && flags != 0) qw::fail(QWGPU_EINVALID_ARG, "ip field '%s' is indexed `basic`, without fieldnorms", name);
  if (flags & QW_FIELD_HAS_FIELDNORMS) {
    if (!fieldnorm_ids) qw::fail(QWGPU_EINVALID_ARG, "field '%s' declares fieldnorms but none given", name);
    f.fieldnorms.assign(fieldnorm_ids, fieldnorm_ids + b->num_docs);
  }
  b->fields.push_back(std::move(f));
  return (int)b->fields.size() - 1;
  QW_API_END
}

int qwgpu_imgb_add_term(qwgpu_imgb* b, uint32_t field_id, const uint8_t* term, uint32_t term_len,
                        const uint32_t* docs, const uint32_t* tfs, uint32_t n) {
  QW_API_BEGIN
  qw::add_term(b, field_id, term, term_len, docs, tfs, n);
  return 0;
  QW_API_END
}

int qwgpu_imgb_add_term_positions(qwgpu_imgb* b, uint32_t field_id, const uint8_t* term, uint32_t term_len,
                                  const uint32_t* docs, const uint32_t* tfs, uint32_t n, const uint32_t* positions, uint64_t n_positions) {
  QW_API_BEGIN
  qw::add_term(b, field_id, term, term_len, docs, tfs, n, positions, n_positions);
  return 0;
  QW_API_END
}

int qwgpu_imgb_add_column(qwgpu_imgb* b, const char* name, uint32_t type, uint32_t cardinality,
                          const uint64_t* values, uint64_t num_vals, const uint32_t* index,
                          const uint8_t* dict_bytes, const uint32_t* dict_offs, uint32_t dict_n) {
  QW_API_BEGIN
  qw::add_column(b, name, type, cardinality, values, num_vals, index, dict_bytes, dict_offs, dict_n);
  return 0;
  QW_API_END
}

int qwgpu_imgb_finish(qwgpu_imgb* b, uint8_t** img, uint64_t* img_len) {
  QW_API_BEGIN
  qw::finish(b, img, img_len);
  return 0;
  QW_API_END
}

int qwgpu_synth_split(const qwgpu_synth_spec* spec, uint8_t** img, uint64_t* img_len) {
  QW_API_BEGIN
  qw::synth_split(spec, img, img_len);
  return 0;
  QW_API_END
}

uint8_t qwgpu_fieldnorm_to_id(uint32_t fieldnorm) { return qw::fieldnorm_to_id(fieldnorm); }
uint32_t qwgpu_id_to_fieldnorm(uint8_t id) { return qw::id_to_fieldnorm(id); }

}  // extern "C"
