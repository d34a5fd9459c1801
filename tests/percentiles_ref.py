"""The percentiles aggregation restated from the documents' values: a Python DDSketch with the reference's default
configuration, the boundary table of a column by brute force over its raw values, and the hashed entries a split's
plan produces (brute force over every doc), without calling the product's mapping.

DDSketch (alpha = 0.01, 2048 bins per store, min_value = 1e-9): key(v) = ceil(ln(v) / ln_1p(2a / (1 - a))) for
v > 1e-9, the key of |v| in a negative store for v < -1e-9, the zero count otherwise; the representative value of key k
is exp(k * gamma_ln) * (2 / (1 + gamma)). Bins are numbered in value order (ordinals): 0 = the zero count,
k - k0 + 1 = positive key k, -(k - k0 + 1) = negative key k, k0 = the key of the smallest double above 1e-9. A
percentiles entry's key is its ordinal minus the ordinal of the column's minimum."""
from __future__ import annotations

import math
import struct
from typing import Dict, List, Optional, Sequence, Tuple

from quickwit_b200 import ffi
from agg_ref import NO_MIN, Cell, Column, mapped_to_f64

ALPHA, MIN_VALUE, MAX_BINS = 0.01, 1e-9, 2048
GAMMA = 1 + 2 * ALPHA / (1 - ALPHA)
GAMMA_LN = math.log1p(2 * ALPHA / (1 - ALPHA))
DEFAULT_PERCENTS = [1.0, 5.0, 25.0, 50.0, 75.0, 95.0, 99.0]


def key(v: float) -> int:
    k = math.ceil(math.log(v) / GAMMA_LN)
    return max(-(1 << 31), min((1 << 31) - 1, k))


K0 = key(math.nextafter(MIN_VALUE, math.inf))


def ordinal(v: float) -> int:
    if v > MIN_VALUE:
        return key(v) - K0 + 1
    if v < -MIN_VALUE:
        return -(key(-v) - K0 + 1)
    return 0


def value(k: int) -> float:
    return math.exp(k * GAMMA_LN) * (2 / (1 + GAMMA))


def f64_bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


class Sketch:
    """Counts per ordinal, the exact minimum and maximum."""

    def __init__(self):
        self.bins: Dict[int, int] = {}
        self.count, self.min, self.max = 0, math.inf, -math.inf

    def add(self, v: float, n: int = 1):
        o = ordinal(v)
        self.bins[o] = self.bins.get(o, 0) + n
        self.count += n
        self.min, self.max = min(self.min, v), max(self.max, v)

    def merge(self, other: "Sketch"):
        for o, n in other.bins.items():
            self.bins[o] = self.bins.get(o, 0) + n
        self.count += other.count
        self.min, self.max = min(self.min, other.min), max(self.max, other.max)

    def collapsed(self) -> "Sketch":
        """Each store keeps its top 2048 keys: keys below (largest key - 2047) count in that key's bin."""
        s = Sketch()
        s.count, s.min, s.max = self.count, self.min, self.max
        for sign in (1, -1):
            keys = {abs(o) + K0 - 1: n for o, n in self.bins.items() if o * sign > 0}
            if not keys:
                continue
            floor_key = max(keys) - (MAX_BINS - 1)
            for k, n in keys.items():
                o = sign * (max(k, floor_key) - K0 + 1)
                s.bins[o] = s.bins.get(o, 0) + n
        if 0 in self.bins:
            s.bins[0] = self.bins[0]
        return s

    def quantile(self, q: float) -> Optional[float]:
        if self.count == 0:
            return None
        if q == 0:
            return self.min
        if q == 1:
            return self.max
        rank = int(q * (self.count - 1))
        run = 0
        for o in sorted(self.bins):
            run += self.bins[o]
            if run > rank:
                return 0.0 if o == 0 else math.copysign(value(abs(o) + K0 - 1), o)
        raise AssertionError("rank beyond the sketch")


def column_f64(col: Column, raw: int) -> float:
    return mapped_to_f64(col.ctype, col.min + col.gcd * raw)


def table_bruteforce(col: Column) -> Tuple[int, List[int]]:
    """(ordinal of index 0, edges): every raw value of the column's range visited in turn (small columns only)."""
    if col.num_vals == 0:
        return 0, []
    max_raw = (int(col.arr.max()) - col.min) // col.gcd
    ords = [ordinal(column_f64(col, r)) for r in range(max_raw + 1)]
    lo, edges = ords[0], [0]
    for r, o in enumerate(ords):
        assert o >= lo + len(edges) - 1, f"bins not monotone at raw {r}"
        while o >= lo + len(edges):
            edges.append(r)
    return lo, edges


def first_ordinal(col: Column) -> int:
    return ordinal(column_f64(col, 0))


def num_bins(col: Optional[Column]) -> int:
    if col is None or col.num_vals == 0:
        return 0
    return ordinal(mapped_to_f64(col.ctype, int(col.arr.max()))) - first_ordinal(col) + 1


# ---- the hashed entries of a plan ------------------------------------------------------------------------------
def plan_nodes(plan: bytes) -> List[ffi.QwAggNode]:
    h = ffi.QwPlanHeader.from_buffer_copy(plan)
    off = ffi.C.sizeof(ffi.QwPlanHeader) + h.num_nodes * ffi.C.sizeof(ffi.QwPlanNode)
    return [ffi.QwAggNode.from_buffer_copy(plan, off + i * ffi.C.sizeof(ffi.QwAggNode)) for i in range(h.num_aggs)]


def entries(plan: bytes, cols: Dict[int, Column], docs: Optional[Sequence[int]] = None) -> Dict[tuple, Cell]:
    """{(node, parent path, key, missing): Cell} of the plan's aggregation tree (terms, histogram and percentiles
    nodes) over the matched docs (None: every doc), in hashed_ref's path form. A percentiles entry: count = values in
    the bin, min / max = their mapped extremes; the `missing` entry counts docs without a value."""
    nodes = plan_nodes(plan)

    def col_of(n):
        return cols.get(n.column) if n.column != ffi.ABSENT else None

    def keys(i: int, d: int) -> List[Tuple[int, bool, int]]:
        n, col = nodes[i], col_of(nodes[i])
        vals = col.doc_values(d) if col is not None else []
        if n.kind == ffi.AGG_TERMS:
            return [(col.raw(v), False, v) for v in vals] or ([(0, True, 0)] if n.has_missing else [])
        if n.kind == ffi.AGG_HISTOGRAM:
            out = []
            for v in vals:
                x = mapped_to_f64(col.ctype, v)
                if n.has_bounds and not (n.bound_min <= x <= n.bound_max):
                    continue
                out.append((math.floor((x - n.offset) / n.interval) - n.base_pos, False, v))
            return out
        assert n.kind == ffi.AGG_PERCENTILES, n.kind
        if not vals:
            return [(0, True, 0)] if n.has_missing else []
        lo = first_ordinal(col)
        return [(ordinal(mapped_to_f64(col.ctype, v)) - lo, False, v) for v in vals]

    out: Dict[tuple, Cell] = {}

    def visit(i: int, d: int, path: tuple):
        for k, miss, v in keys(i, d):
            c = out.setdefault((i, path, k, miss), Cell())
            c.count += 1
            if nodes[i].kind == ffi.AGG_PERCENTILES and not miss:
                c.min, c.max = min(c.min, v), max(c.max, v)
            n = nodes[i]
            for ch in range(n.first_child, n.first_child + n.num_children):
                visit(ch, d, path + ((i, k, miss),))

    num_docs = max(c.num_docs for c in cols.values())
    for d in (range(num_docs) if docs is None else docs):
        for i, n in enumerate(nodes):
            if n.parent == ffi.ABSENT:
                visit(i, int(d), ())
    return out


def as_entry_list(want: Dict[tuple, Cell]) -> List[tuple]:
    """Engine-style entries (node, parent entry, key, flags, (count, sum_bits, min, max)), parents first."""
    order = sorted(want, key=lambda p: len(p[1]))
    index: Dict[tuple, int] = {}
    outl: List[tuple] = []
    for p in order:
        node, path, k, miss = p
        parent = ffi.AGG_NO_PARENT
        if path:
            (pn, pk, pm), up = path[-1], path[:-1]
            parent = index[(pn, up, pk, pm)]
        c = want[p]
        index[p] = len(outl)
        outl.append((node, parent, k, ffi.AGG_ENTRY_MISSING if miss else 0, (c.count, 0, c.min, c.max)))
    return outl


def sketch_of(values: Sequence[float]) -> Sketch:
    s = Sketch()
    for v in values:
        s.add(v)
    return s


def rust_display(x: float) -> str:
    """Rust's f64 Display: shortest round-trip digits, no exponent, no ".0" on whole numbers."""
    r = repr(float(x))
    if "e" in r or "E" in r:
        from decimal import Decimal
        r = format(Decimal(r), "f")
    return r[:-2] if r.endswith(".0") else r


def expected_values(s: Sketch, percents: Sequence[float] = DEFAULT_PERCENTS, keyed: bool = True):
    c = s.collapsed()
    vals = [c.quantile(p / 100) for p in percents]
    if keyed:
        return {rust_display(p): v for p, v in zip(percents, vals)}
    return [{"key": float(p), "value": v} for p, v in zip(percents, vals)]


__all__ = ["Sketch", "table_bruteforce", "entries", "as_entry_list", "num_bins", "first_ordinal", "ordinal", "value",
           "expected_values", "sketch_of", "f64_bits", "NO_MIN"]
