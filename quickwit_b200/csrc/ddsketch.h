// ddsketch.h — the DDSketch behind the percentiles aggregation, host only: the key of a value, the representative
// value of a key, the boundary table of a column, the collapse and the quantile walk. The engine (boundary tables)
// and aggs.cpp (sketches, merges, finalisation) both use it; nothing else restates these formulas.
//
// The reference's percentiles collector adds every value, as f64, to a `sketches-ddsketch` DDSketch with the
// default configuration: relative accuracy alpha = 0.01, at most 2048 bins per store, min_value = 1e-9 (DESIGN.md §2
// lists which of the rules below the REST golden pins).
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <map>
#include <vector>

#include "common.h"

namespace qw {
namespace dds {

constexpr double kAlpha = 0.01;
constexpr double kMinValue = 1e-9;
constexpr int32_t kMaxBins = 2048;
// largest boundary table a column may need: an f64 column over the whole double range spans ~73 000 bins; a
// column holding +-inf would need ~2^32 (Rust's saturating `as i32` of an infinite key)
constexpr int64_t kMaxTableBins = 1 << 17;

inline double gamma() { return 1.0 + 2.0 * kAlpha / (1.0 - kAlpha); }
inline double gamma_ln() { return std::log1p(2.0 * kAlpha / (1.0 - kAlpha)); }

// key of v > min_value: ceil(ln(v) / gamma_ln), converted as Rust's `as i32` (saturating; NaN -> 0)
inline int32_t key(double v) {
  const double k = std::ceil(std::log(v) / gamma_ln());
  if (std::isnan(k)) return 0;
  if (k >= 2147483647.0) return INT32_MAX;
  if (k <= -2147483648.0) return INT32_MIN;
  return (int32_t)k;
}
// representative value of key k: exp(k * gamma_ln) * 2 / (1 + gamma)
inline double value(int32_t k) { return std::exp((double)k * gamma_ln()) * (2.0 / (1.0 + gamma())); }

// Bin ordinals: one integer per (store, key), increasing with the value — the negative store from its largest key
// (the most negative values) down, the zero count (|v| <= min_value) = 0, then the positive store in ascending key
// order. Keys start at the key of the smallest double above min_value, so ordinals are contiguous.
inline int64_t first_key() {
  static const int32_t k = key(std::nextafter(kMinValue, INFINITY));
  return k;
}
inline int64_t bin_ord(double v) {
  if (v > kMinValue) return (int64_t)key(v) - first_key() + 1;
  if (v < -kMinValue) return -((int64_t)key(-v) - first_key() + 1);
  return 0;  // (NaN too: it compares false both ways)
}
// the store (-1 negative, 0 zero count, 1 positive) and key of an ordinal
inline int ord_store(int64_t o) { return o < 0 ? -1 : (o > 0 ? 1 : 0); }
inline int32_t ord_key(int64_t o) { return (int32_t)((o < 0 ? -o : o) + first_key() - 1); }

// Boundary table of a column in raw space: the bins ord_lo .. ord_lo + edges.size() - 1 between the bins of the
// column's minimum and maximum, empty ones included; edges[i] = the smallest raw value whose bin is >= ord_lo + i
// (edges[0] = 0). bin_ord(qw_mapped_to_f64(min + gcd * raw)) is monotone in raw, so each edge is a binary search
// (first_raw), with the same `log` the reference's f64::ln calls. The device finds a raw value's bin as the last edge
// <= raw, and never evaluates a logarithm.
struct Table {
  int64_t ord_lo = 0;
  uint64_t num_bins = 0;
  std::vector<uint64_t> edges;  // (empty unless asked for)
};
// false when the column cannot be tabled: NaN values (they break the order of the bins) or a span of more than
// kMaxTableBins bins (infinite values). A column without values has no bins.
inline bool column_table(const QwImgColumn& c, bool with_edges, Table* t) {
  *t = Table();
  if (!c.num_vals) return true;
  const uint64_t gcd = c.gcd ? c.gcd : 1, max_raw = (c.max_value - c.min_value) / gcd;
  auto ord = [&](uint64_t raw) { return bin_ord(qw_mapped_to_f64(c.type, c.min_value + gcd * raw)); };
  if (std::isnan(qw_mapped_to_f64(c.type, c.min_value)) || std::isnan(qw_mapped_to_f64(c.type, c.max_value))) return false;
  const int64_t lo = ord(0), hi = ord(max_raw);
  if (hi - lo + 1 > kMaxTableBins) return false;
  t->ord_lo = lo;
  t->num_bins = (uint64_t)(hi - lo + 1);
  if (!with_edges) return true;
  t->edges.resize(t->num_bins);
  t->edges[0] = 0;
  for (int64_t i = 1; i < (int64_t)t->num_bins; i++)  // (ord(max_raw) = hi >= lo + i)
    t->edges[i] = first_raw(t->edges[i - 1], max_raw, [&](uint64_t raw) { return ord(raw) >= lo + i; });
  return true;
}

// A sketch as counts per bin ordinal plus the exact minimum and maximum (q = 0 and q = 1 return those).
struct Sketch {
  std::map<int64_t, uint64_t> bins;  // ordinal -> count (no zero counts)
  uint64_t count = 0;
  double min = INFINITY, max = -INFINITY;
  void add(int64_t ord, uint64_t n, double lo, double hi) {
    if (!n) return;
    bins[ord] += n;
    count += n;
    min = std::min(min, lo);
    max = std::max(max, hi);
  }
  void merge(const Sketch& o) {
    for (const auto& kv : o.bins) bins[kv.first] += kv.second;
    count += o.count;
    min = std::min(min, o.min);
    max = std::max(max, o.max);
  }
  // Each store keeps at most kMaxBins keys: when a store spans more, every key below (its largest key - 2047) counts
  // in that key's bin
  void collapse() {
    for (int store = -1; store <= 1; store += 2) {
      int32_t kmax = INT32_MIN;
      for (const auto& kv : bins) if (ord_store(kv.first) == store) kmax = std::max(kmax, ord_key(kv.first));
      if (kmax == INT32_MIN) continue;
      const int32_t floor_key = kmax - (kMaxBins - 1);
      uint64_t moved = 0;
      for (auto it = bins.begin(); it != bins.end();) {
        if (ord_store(it->first) == store && ord_key(it->first) < floor_key) { moved += it->second; it = bins.erase(it); }
        else ++it;
      }
      if (moved) bins[store * ((int64_t)floor_key - first_key() + 1)] += moved;
    }
  }
  // quantile q (0 <= q <= 1) of the sketch as it stands; false when it is empty. rank = floor(q * (count - 1)); the
  // answer is the representative value of the first bin, in value order, whose running count exceeds the rank
  bool quantile(double q, double* out) const {
    if (!count) return false;
    if (q == 0.0) { *out = min; return true; }
    if (q == 1.0) { *out = max; return true; }
    const uint64_t rank = (uint64_t)(q * (double)(count - 1));
    uint64_t run = 0;
    for (const auto& kv : bins) {
      run += kv.second;
      if (run > rank) {
        const int s = ord_store(kv.first);
        *out = s == 0 ? 0.0 : (s > 0 ? value(ord_key(kv.first)) : -value(ord_key(kv.first)));
        return true;
      }
    }
    *out = max;  // (not reached: the bins hold `count` values)
    return true;
  }
};

}  // namespace dds
}  // namespace qw
