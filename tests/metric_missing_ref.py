"""The `missing` parameter of the stats family (stats, avg, sum, min, max, value_count) restated without the product's
value mapping: what the device reports for a split (each stats cell, and under every parent bucket the count of matched
docs without a value as an entry with missing = True, key 0 — or in the dense layout a second bank of cells after the
node's first), and the finalised metric of a set of documents, brute force over their values.

A document without a value in the field counts as the `missing` value exactly once per parent bucket it lands in; a
document with values contributes only those. Values are compared in the space the column's values take as f64 (u64 /
i64 as integers, datetime as nanoseconds, bool as 0 / 1), where `missing` is taken as given."""
from __future__ import annotations

import math
import struct
from fractions import Fraction
from typing import Dict, List, Optional, Sequence

from quickwit_b200 import ffi, plan as P
from agg_ref import U, Cell, Column, _layout, cells
from hashed_ref import _keys, sparse_cells


def _col_of(a: P.Agg, cols: Dict[int, Column]) -> Optional[Column]:
    return cols.get(a.column) if a.column != ffi.ABSENT else None


def missing_entries(aggs: Sequence[P.Agg], cols: Dict[int, Column], docs: Optional[Sequence[int]] = None) -> Dict[tuple, Cell]:
    """{(node, parent path, 0, True): Cell(count = docs without a value)} of every STATS node with `missing`, in
    hashed_ref's path form, over the matched docs `docs` (None: every doc)."""
    lay = _layout(aggs)
    index = {id(a): i for i, (a, _p, _b, _n) in enumerate(lay)}
    out: Dict[tuple, Cell] = {}

    def visit(a: P.Agg, d: int, path: tuple):
        i, col = index[id(a)], _col_of(a, cols)
        if a.kind == ffi.AGG_STATS:
            if a.missing is not None and not (col.doc_values(d) if col is not None else []):
                out.setdefault((i, path, 0, True), Cell()).count += 1
            return
        for key, miss in _keys(a, col, d):
            for ch in a.children:
                visit(ch, d, path + ((i, key, miss),))

    num_docs = max(c.num_docs for c in cols.values())
    for d in (range(num_docs) if docs is None else docs):
        for a in aggs:
            visit(a, int(d), ())
    return out


def device_entries(aggs: Sequence[P.Agg], cols: Dict[int, Column], docs: Optional[Sequence[int]] = None) -> Dict[tuple, Cell]:
    """The hashed layout's entries of a split: hashed_ref.sparse_cells and the `missing` counts."""
    out = sparse_cells(aggs, cols, docs)
    out.update(missing_entries(aggs, cols, docs))
    return out


def dense_cells(aggs: Sequence[P.Agg], cols: Dict[int, Column], docs: Optional[Sequence[int]] = None) -> List[Cell]:
    """The dense layout of a split: agg_ref.cells with, after the cells of every STATS node with `missing`, one cell
    per parent cell holding the count of docs without a value."""
    lay = _layout(aggs)
    base_cells = cells(aggs, cols, docs)
    miss = missing_entries(aggs, cols, docs)
    out: List[Cell] = []
    for i, (a, p, base, n) in enumerate(lay):
        out.extend(base_cells[base:base + n])
        if a.kind == ffi.AGG_STATS and a.missing is not None:
            bank = [Cell() for _ in range(n)]
            for (node, path, _k, _m), c in miss.items():
                if node == i:
                    bank[_parent_cell(lay, path)].count = c.count
            out.extend(bank)
    return out


def _parent_cell(lay, path: tuple) -> int:
    """Row-major index of a parent path ((node, key, missing), ...) among the parent's cells (a terms `missing`
    bucket is the node's last)."""
    cell = 0
    for node, key, miss in path:
        a = lay[node][0]
        cell = cell * a.num_buckets + (a.num_buckets - 1 if miss else key)
    return cell


# ---- the finalised metric, brute force over the documents' values ----------------------------------------------
class Expect:
    """A metric over a bag of values (Python ints for integer columns, floats for f64 ones) and n docs without a value
    that count as `missing`."""

    def __init__(self, vals: Sequence, n_missing: int = 0, missing: Optional[float] = None):
        self.vals, self.n, self.m = list(vals), n_missing if missing is not None else 0, missing
        self.count = len(self.vals) + self.n
        pts = [float(v) for v in self.vals] + ([float(missing)] if self.n else [])
        self.min = min(pts) if pts else None
        self.max = max(pts) if pts else None
        self.exact_sum = sum((Fraction(v) for v in self.vals), Fraction(0)) + (self.n * Fraction(missing) if self.n else 0)
        # recursive summation in any order, the n * missing product and the merge of up to a few splits stay within
        # γ(k) Σ|v| with k = values + 4
        k = (len(self.vals) + 4) * U
        self.sum_tol = k / (1 - k) * (math.fsum(abs(float(v)) for v in self.vals) + (self.n * abs(float(missing)) if self.n else 0.0))

    def sum_ok(self, got: float, exact: bool) -> bool:
        want = float(self.exact_sum)
        return got == want if exact else abs(got - want) <= self.sum_tol

    def check(self, kind: str, got, exact: bool = False, ctx: str = ""):
        """got: the finalised JSON of a metric of `kind` (stats / avg / sum / min / max / value_count)."""
        some = self.count > 0
        if kind == "stats":
            assert got["count"] == self.count, f"{ctx}: count {got['count']} != {self.count}"
            assert (got["min"], got["max"]) == (self.min, self.max), f"{ctx}: min/max {(got['min'], got['max'])} != {(self.min, self.max)}"
            assert self.sum_ok(got["sum"], exact), f"{ctx}: sum {got['sum']!r} vs {float(self.exact_sum)!r} (tol {self.sum_tol!r})"
            self._avg(got["avg"], exact, ctx)
        elif kind == "value_count":
            assert got["value"] == float(self.count), f"{ctx}: value_count {got['value']} != {self.count}"
        elif kind == "min":
            assert got["value"] == self.min, f"{ctx}: min {got['value']} != {self.min}"
        elif kind == "max":
            assert got["value"] == self.max, f"{ctx}: max {got['value']} != {self.max}"
        elif kind == "sum":
            assert self.sum_ok(got["value"], exact), f"{ctx}: sum {got['value']!r} vs {float(self.exact_sum)!r}"
        else:
            assert kind == "avg", kind
            self._avg(got["value"], exact, ctx)
        assert some or kind in ("sum", "value_count", "stats") or got["value"] is None, ctx

    def _avg(self, got, exact: bool, ctx: str):
        if not self.count:
            assert got is None, f"{ctx}: avg {got} of nothing"
            return
        want = float(self.exact_sum) / self.count if exact else float(self.exact_sum / self.count)
        tol = 0.0 if exact else self.sum_tol / self.count + abs(want) * 2 * U
        assert abs(got - want) <= tol, f"{ctx}: avg {got!r} vs {want!r} (tol {tol!r})"



# ---- documents, and the finalised aggregation tree checked bucket by bucket -----------------------------------------
TYPES = ("u64", "i64", "f64", "datetime", "bool")
CARDS = ("full", "optional", "multi", "absent")
FIELDS = [f"{t}_{c}" for t in TYPES for c in CARDS]
HOUR_S = 3600


def mapping(with_absent: bool = True) -> dict:
    """g: terms key (u64), ts: datetime (seconds), h: i64 histogram key, and one value field per (type, cardinality);
    the `absent` fields are left out of the mapping of the split that lacks them."""
    fm = [{"name": "g", "type": "u64", "fast": True}, {"name": "ts", "type": "datetime", "fast": True},
          {"name": "h", "type": "i64", "fast": True}]
    fm += [{"name": f, "type": f.split("_")[0], "fast": True} for f in FIELDS if with_absent or not f.endswith("_absent")]
    return {"field_mappings": fm, "timestamp_field": "ts"}


def _value(t: str, rng):
    if t == "u64":
        return int(rng.integers(0, 1000))
    if t == "i64":
        return int(rng.integers(-500, 500))
    if t == "f64":
        return float(rng.normal(0, 100))
    if t == "datetime":
        return int(rng.integers(1_700_000_000, 1_700_000_000 + 86_400))
    return bool(rng.integers(0, 2))


def make_docs(n: int, rng, absent: bool = False) -> List[dict]:
    """n documents: `full` fields hold one value, `optional` none in about 30 % of docs, `multi` 0, 1 or 3; `absent`
    fields like `optional`, or nothing when `absent` (the split built without them)."""
    docs = []
    for _ in range(n):
        d = {"g": int(rng.integers(0, 4)), "ts": int(1_700_000_000 + rng.integers(0, 6 * HOUR_S)), "h": int(rng.integers(-40, 40))}
        for f in FIELDS:
            t, c = f.split("_")
            if c == "full":
                d[f] = _value(t, rng)
            elif c == "multi":
                k = int(rng.choice([0, 1, 3]))
                if k:
                    d[f] = [_value(t, rng) for _ in range(k)]
            elif not (c == "absent" and absent) and rng.random() >= 0.3:
                d[f] = _value(t, rng)
        docs.append(d)
    return docs


def f64_space(field: str, v):
    """A document value as the column's values read in f64 space: integers stay exact ints, datetimes are nanoseconds."""
    t = field.split("_")[0]
    if t == "datetime":
        return int(v) * 10**9
    if t == "bool":
        return int(bool(v))
    return v


def doc_values(d: dict, field: str) -> list:
    x = d.get(field)
    return [f64_space(field, v) for v in (x if isinstance(x, list) else ([] if x is None else [x]))]


def expect(docs: Sequence[dict], field: str, missing: Optional[float]) -> Expect:
    vals, n = [], 0
    for d in docs:
        vs = doc_values(d, field)
        vals += vs
        n += not vs
    return Expect(vals, n, missing)


METRICS = ("stats", "avg", "sum", "min", "max", "value_count")


def _bucket_docs(kind: str, spec: dict, docs: Sequence[dict], key) -> List[dict]:
    f = spec["field"]
    if kind == "terms":
        return [d for d in docs if d.get(f) == key]
    if kind == "date_histogram":
        step = 3_600_000  # fixed_interval 1h, keys in ms
        return [d for d in docs if (d[f] * 1000) // step * step == key]
    iv = spec["interval"]
    return [d for d in docs if math.floor(d[f] / iv) * iv == key]


def check_tree(req: dict, got: dict, docs: Sequence[dict], exact: bool = False, ctx: str = ""):
    """Every metric of the finalised result `got` of request `req` against the brute force over `docs` (bucket keys
    from the request's terms / date_histogram / histogram on single-valued fields, doc counts included)."""
    for name, body in req.items():
        kind = next(k for k in body if k != "aggs")
        spec, r = body[kind], got[name]
        c = f"{ctx}/{name}"
        if kind in METRICS:
            expect(docs, spec["field"], spec.get("missing")).check(kind, r, exact, c)
            continue
        keys = set()
        for b in r["buckets"]:
            sub = _bucket_docs(kind, spec, docs, b["key"])
            assert b["doc_count"] == len(sub), f"{c}[{b['key']}]: doc_count {b['doc_count']} != {len(sub)}"
            keys.add(b["key"])
            if "aggs" in body:
                check_tree(body["aggs"], b, sub, exact, f"{c}[{b['key']}]")
        if kind == "terms":
            assert keys == {d[spec["field"]] for d in docs}, f"{c}: bucket keys {sorted(keys)}"
            order = spec.get("order")
            if order:
                (target, direction), = order.items()
                sub_spec = next(v for k, v in body["aggs"][target].items())
                avg = {k: expect(_bucket_docs(kind, spec, docs, k), sub_spec["field"], sub_spec.get("missing")) for k in keys}
                val = {k: float(e.exact_sum) / e.count if e.count else 0.0 for k, e in avg.items()}
                want = sorted(keys, key=lambda k: (-val[k] if direction == "desc" else val[k], k))
                assert [b["key"] for b in r["buckets"]] == want, f"{c}: order {[b['key'] for b in r['buckets']]} != {want}"


def request(field: str, missing, levels=("top", "terms", "date_histogram", "terms_histogram"), kinds=METRICS) -> dict:
    """Each metric kind over `field` with `missing` (None: without), at each of `levels`."""
    def metrics(suffix):
        out = {}
        for k in kinds:
            spec = {"field": field}
            if missing is not None:
                spec["missing"] = missing
            out[f"{k}{suffix}"] = {k: spec}
        return out

    req = {}
    if "top" in levels:
        req.update(metrics(""))
    if "terms" in levels:
        req["by_g"] = {"terms": {"field": "g"}, "aggs": metrics("_g")}
    if "date_histogram" in levels:
        req["by_hour"] = {"date_histogram": {"field": "ts", "fixed_interval": "1h"}, "aggs": metrics("_t")}
    if "terms_histogram" in levels:
        req["by_g_h"] = {"terms": {"field": "g"}, "aggs": {"by_h": {"histogram": {"field": "h", "interval": 10}, "aggs": metrics("_h")}}}
    return req


# ---- between the compiled plan, the restated entries and the leaf builder ---------------------------------------------
def aggs_from_plan(plan: bytes) -> List[P.Agg]:
    """The compiled plan's aggregation nodes as P.Agg trees (the top-level nodes), for the restatements above."""
    h = ffi.QwPlanHeader.from_buffer_copy(plan)
    off = ffi.C.sizeof(ffi.QwPlanHeader) + h.num_nodes * ffi.C.sizeof(ffi.QwPlanNode)
    nodes = [ffi.QwAggNode.from_buffer_copy(plan, off + i * ffi.C.sizeof(ffi.QwAggNode)) for i in range(h.num_aggs)]
    aggs = [P.Agg(n.kind, column=n.column, num_buckets=n.num_buckets, interval=n.interval, offset=n.offset, base_pos=n.base_pos,
                  bounds=(n.bound_min, n.bound_max) if n.has_bounds else None,
                  ranges=[(n.range_from[r], n.range_to[r]) for r in range(n.num_ranges)],
                  missing=n.missing_value if n.has_missing else None) for n in nodes]
    for a, n in zip(aggs, nodes):
        a.children = aggs[n.first_child:n.first_child + n.num_children]
    return [a for a, n in zip(aggs, nodes) if n.parent == ffi.ABSENT]


def cell_tuple(c: Cell) -> tuple:
    """(count, sum_bits, min_mapped, max_mapped) of a restated cell: the exact raw sum, or the f64 bits of fsum."""
    if c.sum is None:
        s = 0
    elif c.sum.exact:
        s = c.sum.raw
    else:
        s = struct.unpack("<Q", struct.pack("<d", c.sum.fsum()))[0]
    return (c.count, s, c.min, c.max)


def as_entry_list(want: Dict[tuple, Cell]) -> List[tuple]:
    """Engine-style entries (node, parent entry, key, flags, cell) of restated paths, parents first."""
    index: Dict[tuple, int] = {}
    out: List[tuple] = []
    for p in sorted(want, key=lambda p: len(p[1])):
        node, path, k, miss = p
        parent = ffi.AGG_NO_PARENT
        if path:
            (pn, pk, pm), up = path[-1], path[:-1]
            parent = index[(pn, up, pk, pm)]
        index[p] = len(out)
        out.append((node, parent, k, ffi.AGG_ENTRY_MISSING if miss else 0, cell_tuple(want[p])))
    return out
