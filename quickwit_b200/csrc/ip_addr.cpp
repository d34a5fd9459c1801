// ip_addr.cpp — parser and printer of `ip` field values (declarations and contract in ip_addr.h).
//
// The parser follows Rust std's core::net::parser step by step: every reader works on a cursor and restores it when
// it fails (read_atomically), so a dotted IPv4 tail that does not parse falls back to a hex group exactly as there.
#include "ip_addr.h"

#include <cstdio>
#include <cstring>

#include "common.h"

namespace qw {
namespace {

struct Parser {
  const char* p;
  const char* e;

  int peek() const { return p < e ? (unsigned char)*p : -1; }
  bool read_given_char(char c) {
    if (p < e && *p == c) { p++; return true; }
    return false;
  }
  static int digit(int c, uint32_t radix) {
    int d = -1;
    if (c >= '0' && c <= '9') d = c - '0';
    else if (c >= 'a' && c <= 'z') d = c - 'a' + 10;
    else if (c >= 'A' && c <= 'Z') d = c - 'A' + 10;
    return d >= 0 && (uint32_t)d < radix ? d : -1;
  }
  // read_number(radix, Some(max_digits), allow_zero_prefix) into a value of at most `max_value`
  bool read_number(uint32_t radix, int max_digits, bool allow_zero_prefix, uint32_t max_value, uint32_t* out) {
    const char* start = p;
    const bool has_leading_zero = peek() == '0';
    uint32_t v = 0;
    int count = 0;
    for (int d; (d = digit(peek(), radix)) >= 0;) {
      p++;
      v = v * radix + (uint32_t)d;  // max_digits keeps this far below overflow
      if (v > max_value || ++count > max_digits) { p = start; return false; }
    }
    if (count == 0 || (!allow_zero_prefix && has_leading_zero && count > 1)) { p = start; return false; }
    *out = v;
    return true;
  }
  bool read_ipv4(uint8_t o[4]) {
    const char* start = p;
    for (int i = 0; i < 4; i++) {
      uint32_t v;
      if ((i > 0 && !read_given_char('.')) || !read_number(10, 3, false, 255, &v)) { p = start; return false; }
      o[i] = (uint8_t)v;
    }
    return true;
  }
  // read_groups: up to `limit` groups; *ipv4 when the last two came from a dotted tail
  int read_groups(uint16_t* groups, int limit, bool* ipv4) {
    *ipv4 = false;
    for (int i = 0; i < limit; i++) {
      if (i < limit - 1) {  // a trailing embedded IPv4 address needs two groups
        const char* start = p;
        uint8_t o[4];
        if ((i == 0 || read_given_char(':')) && read_ipv4(o)) {
          groups[i] = (uint16_t)(o[0] << 8 | o[1]);
          groups[i + 1] = (uint16_t)(o[2] << 8 | o[3]);
          *ipv4 = true;
          return i + 2;
        }
        p = start;
      }
      const char* start = p;
      uint32_t g;
      if (!((i == 0 || read_given_char(':')) && read_number(16, 4, true, 0xFFFF, &g))) { p = start; return i; }
      groups[i] = (uint16_t)g;
    }
    return limit;
  }
  bool read_ipv6(uint16_t seg[8]) {
    const char* start = p;
    memset(seg, 0, 16);
    bool head_ipv4;
    const int head = read_groups(seg, 8, &head_ipv4);
    if (head == 8) return true;
    if (head_ipv4 || !read_given_char(':') || !read_given_char(':')) { p = start; return false; }  // no IPv4 before `::`
    uint16_t tail[7] = {0};
    bool tail_ipv4;
    const int n = read_groups(tail, 8 - (head + 1), &tail_ipv4);  // `::` stands for at least one zero group
    for (int i = 0; i < n; i++) seg[8 - n + i] = tail[i];
    return true;
  }
};

}  // namespace

bool parse_ip_addr(const char* s, size_t n, uint8_t out[16]) {
  Parser ps{s, s + n};
  uint8_t v4[4];
  if (ps.read_ipv4(v4)) {  // IpAddr::V4, then into_ipv6_addr: ::ffff:a.b.c.d
    if (ps.p != ps.e) return false;
    memset(out, 0, 10);
    out[10] = out[11] = 0xFF;
    memcpy(out + 12, v4, 4);
    return true;
  }
  uint16_t seg[8];
  if (!ps.read_ipv6(seg) || ps.p != ps.e) return false;
  for (int i = 0; i < 8; i++) { out[2 * i] = (uint8_t)(seg[i] >> 8); out[2 * i + 1] = (uint8_t)seg[i]; }
  return true;
}

std::string format_ip_addr(const uint8_t a[16]) {
  char buf[48];
  static const uint8_t kMapped[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0xFF, 0xFF};
  if (memcmp(a, kMapped, 12) == 0) {
    snprintf(buf, sizeof buf, "%u.%u.%u.%u", a[12], a[13], a[14], a[15]);
    return buf;
  }
  uint16_t seg[8];
  for (int i = 0; i < 8; i++) seg[i] = (uint16_t)(a[2 * i] << 8 | a[2 * i + 1]);
  int best_start = 0, best_len = 0, cur_start = 0, cur_len = 0;
  for (int i = 0; i < 8; i++) {
    if (seg[i] == 0) {
      if (cur_len == 0) cur_start = i;
      if (++cur_len > best_len) { best_len = cur_len; best_start = cur_start; }
    } else cur_len = 0;
  }
  std::string out;
  auto part = [&](int from, int to) {
    for (int i = from; i < to; i++) {
      if (i > from) out += ':';
      snprintf(buf, sizeof buf, "%x", seg[i]);
      out += buf;
    }
  };
  if (best_len > 1) {
    part(0, best_start);
    out += "::";
    part(best_start + best_len, 8);
  } else part(0, 8);
  return out;
}

}  // namespace qw

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

int qwgpu_parse_ip(const char* text, uint64_t len, uint8_t* out16) {
  QW_API_BEGIN
  if (!qw::parse_ip_addr(text, (size_t)len, out16))
    qw::fail(QWGPU_EINVALID_ARG, "`%.*s` is not an IP address", (int)(len > 64 ? 64 : len), text);
  return 0;
  QW_API_END
}

int qwgpu_format_ip(const uint8_t* addr16, char* out, uint64_t cap) {
  QW_API_BEGIN
  const std::string s = qw::format_ip_addr(addr16);
  if (s.size() + 1 > cap) qw::fail(QWGPU_EINVALID_ARG, "qwgpu_format_ip: buffer of %llu bytes is too small", (unsigned long long)cap);
  memcpy(out, s.c_str(), s.size() + 1);
  return (int)s.size();
  QW_API_END
}

}  // extern "C"
