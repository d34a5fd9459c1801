// ip_addr.h — the text forms of `ip` field values: one parser and one printer for the image builder, the query
// compiler and the aggregation keys.
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>

namespace qw {

// Rust std's `IpAddr::from_str` (core::net::parser) followed by `into_ipv6_addr` (quickwit-query json_literal.rs):
// the whole of s[0, n) must be one address. IPv4: exactly four decimal octets, each <= 255, no leading zeros.
// IPv6: up to eight groups of 1-4 hex digits, at most one `::`, and an optional dotted IPv4 tail in place of the last
// two groups. No zone id, brackets, port or surrounding whitespace. An IPv4 address becomes its IPv4-mapped form
// ::ffff:a.b.c.d. out = the 16 big-endian bytes; false when s is not an address.
bool parse_ip_addr(const char* s, size_t n, uint8_t out[16]);
inline bool parse_ip_addr(const std::string& s, uint8_t out[16]) { return parse_ip_addr(s.data(), s.size(), out); }

// An address as a terms bucket key: the dotted quad when it is IPv4-mapped, else Rust's `Ipv6Addr` Display (RFC
// 5952: lower-case hex without leading zeros, the first longest run of two or more zero groups as `::`).
std::string format_ip_addr(const uint8_t a[16]);

}  // namespace qw
