"""The aggregation value rules the host and the kernels share (device_types.h, common.h, ddsketch.h): a column's mapped
value as f64 (qw_mapped_to_f64), the histogram position floor((val - offset) / interval) (qw_hist_pos), the raw-space
boundary table of a histogram node that the fast aggregation paths search instead of evaluating the position
(hist_bounds), and the percentiles boundary table (dds::column_table). Compiled from the headers with g++ and pinned
against struct-based restatements and brute force, without a GPU."""
import ctypes as C
import math
import os
import struct
import subprocess

import pytest

from quickwit_b200 import ffi, service
from test_percentiles_host import TABLE_COLUMNS, table_split  # noqa: F401  (the fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U64 = (1 << 64) - 1

SHIM = r'''#include "ddsketch.h"
extern "C" double mapped_to_f64(unsigned type, unsigned long long m) { return qw_mapped_to_f64(type, m); }
extern "C" unsigned long long f64_to_mapped(double d) { return f64_to_u64(d); }
extern "C" double hist_pos(double val, double offset, double interval) { return qw_hist_pos(val, offset, interval); }
extern "C" void hist_table(unsigned type, unsigned long long min_value, unsigned long long gcd, unsigned long long max_raw,
                           unsigned has_bounds, double bound_min, double bound_max, double offset, double interval,
                           long long base_pos, unsigned nb, unsigned long long* out) {
  DCol c{};
  c.type = type; c.min_value = min_value; c.gcd = gcd;
  DAgg d{};
  d.kind = QW_AGG_HISTOGRAM; d.num_buckets = nb; d.has_bounds = has_bounds; d.bound_min = bound_min; d.bound_max = bound_max;
  d.offset = offset; d.interval = interval; d.base_pos = base_pos;
  std::vector<uint64_t> v;
  qw::hist_bounds(c, max_raw, d, v);
  memcpy(out, v.data(), v.size() * 8);
}
extern "C" long long pct_table(const uint8_t* img, unsigned long long len, unsigned col, long long* first, unsigned long long* edges,
                               unsigned long long cap) {
  qw::ImageView v;
  v.open(img, len);
  qw::dds::Table t;
  if (!qw::dds::column_table(v.columns[col], true, &t)) return -1;
  *first = t.ord_lo;
  for (size_t i = 0; i < t.edges.size() && i < cap; i++) edges[i] = t.edges[i];
  return (long long)t.num_bins;
}
'''


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("agg_value_rules")
    (d / "shim.cpp").write_text(SHIM)
    cxx = os.environ.get("CXX", "g++")
    subprocess.run([cxx, "-O2", "-Wall", "-Werror", "-std=c++17", "-fno-fast-math", "-ffp-contract=off", "-fPIC", "-shared",
                    "-I", os.path.join(ROOT, "quickwit_b200", "csrc"), "-o", str(d / "shim.so"), str(d / "shim.cpp")], check=True)
    lib = C.CDLL(str(d / "shim.so"))
    lib.mapped_to_f64.restype, lib.mapped_to_f64.argtypes = C.c_double, [C.c_uint, C.c_ulonglong]
    lib.f64_to_mapped.restype, lib.f64_to_mapped.argtypes = C.c_ulonglong, [C.c_double]
    lib.hist_pos.restype, lib.hist_pos.argtypes = C.c_double, [C.c_double] * 3
    lib.hist_table.restype = None
    lib.hist_table.argtypes = [C.c_uint, C.c_ulonglong, C.c_ulonglong, C.c_ulonglong, C.c_uint, C.c_double, C.c_double, C.c_double,
                               C.c_double, C.c_longlong, C.c_uint, C.POINTER(C.c_ulonglong)]
    lib.pct_table.restype = C.c_longlong
    lib.pct_table.argtypes = [C.c_void_p, C.c_ulonglong, C.c_uint, C.POINTER(C.c_longlong), C.POINTER(C.c_ulonglong), C.c_ulonglong]
    return lib


# ---- restatements ------------------------------------------------------------------------------------------------
def bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def from_bits(b: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", b))[0]


def mapped_of(x: float) -> int:
    """tantivy's f64 -> u64: flip every bit of a negative double, the sign bit of any other"""
    b = bits(x)
    return b ^ U64 if b >> 63 else b ^ (1 << 63)


def i64_mapped(v: int) -> int:
    return (v + (1 << 63)) & U64


def f64_of(ctype: int, m: int) -> float:
    if ctype in (ffi.COL_U64, ffi.COL_BOOL, ffi.COL_STR, ffi.COL_IP):  # (str and ip: ordinals)
        return float(m)
    if ctype in (ffi.COL_I64, ffi.COL_DATETIME):
        return float(struct.unpack("<q", struct.pack("<Q", m ^ (1 << 63)))[0])
    return from_bits(m ^ (1 << 63) if m >> 63 else m ^ U64)  # f64 (bytes columns: every aggregation refuses them)


# ---- value mapping -----------------------------------------------------------------------------------------------
SPECIAL_F64 = [0.0, -0.0, math.inf, -math.inf, math.nan, from_bits(0xFFF8000000000001), from_bits(0x7FF0000000000001)]
PATTERNS = [0, 1, 2, (1 << 63) - 1, 1 << 63, (1 << 63) + 1, U64 - 1, U64] + [bits(x) for x in SPECIAL_F64] + \
           [mapped_of(x) for x in SPECIAL_F64]


@pytest.mark.parametrize("ctype", range(8))
def test_mapped_to_f64_of_every_column_type(shim, ctype):
    for m in PATTERNS:
        assert bits(shim.mapped_to_f64(ctype, m)) == bits(f64_of(ctype, m)), (ctype, hex(m))


def test_f64_mapping_round_trips(shim):
    for x in SPECIAL_F64 + [1.5, -1.5, 5e-324, -5e-324, 1.7976931348623157e308, -1.7976931348623157e308]:
        m = shim.f64_to_mapped(x)
        assert m == mapped_of(x), x
        assert bits(shim.mapped_to_f64(ffi.COL_F64, m)) == bits(x), x
    # the mapping keeps the order of the doubles: -inf < -1 < -0.0 < 0.0 < 1 < inf
    order = [-math.inf, -1.0, -5e-324, -0.0, 0.0, 5e-324, 1.0, math.inf]
    assert [shim.f64_to_mapped(x) for x in order] == sorted(shim.f64_to_mapped(x) for x in order)


# ---- histogram position ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("offset,interval", [(0.0, 1.0), (-3.5, 7.0), (2.25, 0.1), (-1e-3, 0.3), (-4 * 86_400e9, 3_600e9),
                                             (0.5, 1e-300), (-7.0, 2.0 ** -20)])
def test_hist_pos_at_bucket_edges(shim, offset, interval):
    for k in [-1000, -3, -2, -1, 0, 1, 2, 3, 17, 1000, 123_456]:
        edge = k * interval + offset
        for v in (math.nextafter(edge, -math.inf), edge, math.nextafter(edge, math.inf)):
            assert shim.hist_pos(v, offset, interval) == float(math.floor((v - offset) / interval)), (v, offset, interval)


# ---- histogram boundary table ------------------------------------------------------------------------------------
def plan_layout(ctype, min_value, gcd, max_raw, offset, interval, hard=None):
    """(base_pos, num_buckets) from the column's smallest and largest value, as the plan compiler lays them out"""
    lo, hi = f64_of(ctype, min_value), f64_of(ctype, min_value + gcd * max_raw)
    if hard:
        lo, hi = max(lo, hard[0]), min(hi, hard[1])
    p0, p1 = math.floor((lo - offset) / interval), math.floor((hi - offset) / interval)
    return p0, p1 - p0 + 1


def bucket(ctype, min_value, gcd, offset, interval, hard, base_pos, nb, raw):
    """bucket of a raw value, clamped to [-1, nb]"""
    val = f64_of(ctype, min_value + gcd * raw)
    if hard and not val >= hard[0]:
        return -1
    if hard and not val <= hard[1]:
        return nb
    return min(max(math.floor((val - offset) / interval) - base_pos, -1), nb)


TABLES = {
    "u64": (ffi.COL_U64, 5, 1, 300, 0.0, 7.0, None),
    "u64_neg_offset": (ffi.COL_U64, 5, 1, 300, -3.5, 7.0, None),
    "u64_gcd": (ffi.COL_U64, 4, 6, 200, 2.5, 10.0, None),
    "u64_gcd_bounds": (ffi.COL_U64, 4, 6, 200, 2.5, 10.0, (100.0, 933.0)),
    "bool": (ffi.COL_BOOL, 0, 1, 1, 0.0, 1.0, None),
    "i64": (ffi.COL_I64, i64_mapped(-500), 3, 400, -7.0, 25.0, None),
    "i64_bounds": (ffi.COL_I64, i64_mapped(-500), 3, 400, -7.0, 25.0, (-301.5, 250.0)),
    "i64_fractional": (ffi.COL_I64, i64_mapped(-50), 1, 100, -0.25, 0.75, None),
    "f64_around_zero": (ffi.COL_F64, mapped_of(-1e-320), 1, 2 * 2024, 0.0, 1e-321, None),
    "f64_around_zero_bounds": (ffi.COL_F64, mapped_of(-1e-320), 1, 2 * 2024, -5e-324, 1e-321, (-3e-321, 4e-321)),
    "f64_gcd": (ffi.COL_F64, mapped_of(1.0), 1 << 40, 1000, 0.005, 0.01, None),
    "f64_negative_gcd": (ffi.COL_F64, mapped_of(-2.0), 1 << 40, 1000, -0.3, 0.05, None),
    "date": (ffi.COL_DATETIME, i64_mapped(1_420_070_400 * 10**9), 10**9, 20_000, -4 * 3_600e9, 3_600e9, None),
    "date_bounds": (ffi.COL_DATETIME, i64_mapped(1_420_070_400 * 10**9), 10**9, 20_000, 0.0, 1_800e9,
                    (1_420_072_000e9, 1_420_080_000e9)),
}


def table(shim, ctype, min_value, gcd, max_raw, offset, interval, hard):
    base_pos, nb = plan_layout(ctype, min_value, gcd, max_raw, offset, interval, hard)
    out = (C.c_ulonglong * (nb + 1))()
    shim.hist_table(ctype, min_value, gcd, max_raw, 1 if hard else 0, hard[0] if hard else 0.0, hard[1] if hard else 0.0,
                    offset, interval, base_pos, nb, out)
    return base_pos, nb, list(out)


@pytest.mark.parametrize("name", list(TABLES))
def test_histogram_table_matches_brute_force(shim, name):
    ctype, min_value, gcd, max_raw, offset, interval, hard = TABLES[name]
    base_pos, nb, edges = table(shim, ctype, min_value, gcd, max_raw, offset, interval, hard)
    assert nb >= 2
    buckets = [bucket(ctype, min_value, gcd, offset, interval, hard, base_pos, nb, r) for r in range(max_raw + 1)]
    want = [next((r for r, b in enumerate(buckets) if b >= k), max_raw + 1) for k in range(nb + 1)]
    assert edges == want
    if hard:  # the bounds cut the column: raws below bound_min lie before edge 0, raws above it past edge nb
        assert buckets[0] == -1 and buckets[-1] == nb


@pytest.mark.parametrize("ctype,offset,interval", [(ffi.COL_U64, 0.0, 2.0 ** 60), (ffi.COL_U64, 3.0, 1e18),
                                                   (ffi.COL_I64, 5e16, 1e17), (ffi.COL_I64, -1.0, 2.0 ** 61)])
def test_histogram_table_over_the_whole_u64_range(shim, ctype, offset, interval):
    """max_raw = 2^64 - 1: the last edge, which no raw value reaches, saturates at 2^64 - 1 instead of 2^64"""
    base_pos, nb, edges = table(shim, ctype, 0, 1, U64, offset, interval, None)
    b = lambda r: bucket(ctype, 0, 1, offset, interval, None, base_pos, nb, r)  # noqa: E731
    assert edges[0] == 0 and edges[nb] == U64 and b(U64) == nb - 1
    for k in range(1, nb):
        e = edges[k]
        assert b(e) >= k and b(e - 1) < k, (k, e)


# ---- percentiles boundary table ----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(TABLE_COLUMNS))
def test_percentiles_table_from_the_headers(shim, table_split, name):  # noqa: F811
    ci = table_split.by_name[name]
    first, edges = service.percentiles_table(table_split.img, ci)
    got_first, buf = C.c_longlong(), (C.c_ulonglong * max(len(edges), 1))()
    assert shim.pct_table(table_split.img.ptr, table_split.img.nbytes, ci, C.byref(got_first), buf, len(edges)) == len(edges)
    assert (got_first.value, list(buf)[:len(edges)]) == (first, edges)
