"""Aggregation requests of 9 to 32 nodes over one corpus shape, for the host and GPU tests of wide plans.

The corpus is built from documents (splitgen.build_split), so the same splits serve seam-C plans and protobuf
requests; `WideSplit` restates every fast field as an agg_ref Column. Fields: FULL columns (svc, lat, code, latf, t and
k00..k47, and the datetime `ts` = t for requests), OPTIONAL ones (opt, optf: a value in most docs, none in the rest) and MULTI ones (lvl, tags: zero to three
values per doc), plus a text field `body` for term queries ranked by _score. Plan builders give flat, two-level and
three-level trees of exactly n nodes in the dense layout, fast-path plans, hashed chains and composites."""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np

from quickwit_b200 import ffi, plan as P, splitgen as S
from agg_corpora import Split
from agg_ref import Column

MAX_NODES, MAX_LEVELS, MAX_AGG_COLUMNS, MAX_QUERY_COLUMNS = 32, 8, 32, 16
QA_MAX_AGGS, QA_MAX_CELLS = 8, 4096
T0 = 1_700_000_000
K_COLS = 48

MAPPING = {"field_mappings": [{"name": "body", "type": "text", "record": "freq", "fieldnorms": True},
                              {"name": "svc", "type": "u64", "fast": True},
                              {"name": "lat", "type": "u64", "fast": True},
                              {"name": "code", "type": "i64", "fast": True},
                              {"name": "latf", "type": "f64", "fast": True},
                              {"name": "t", "type": "i64", "fast": True},
                              {"name": "ts", "type": "datetime", "fast": True, "fast_precision": "seconds"},
                              {"name": "opt", "type": "u64", "fast": True},
                              {"name": "optf", "type": "f64", "fast": True},
                              {"name": "lvl", "type": "u64", "fast": True},
                              {"name": "tags", "type": "u64", "fast": True}] +
           [{"name": f"k{i:02d}", "type": "u64", "fast": True} for i in range(K_COLS)]}
TYPES = {f["name"]: f["type"] for f in MAPPING["field_mappings"]}
WORDS = ("a", "b", "c", "d", "e")


def make_docs(n: int, seed: int) -> List[dict]:
    rng = np.random.default_rng(seed)
    svc, lat, code = rng.integers(0, 8, n), rng.integers(0, 5000, n), rng.integers(-50, 50, n)
    latf, t = rng.normal(10, 30, n), T0 + np.sort(rng.integers(0, 6 * 3600, n))
    opt, optf = rng.integers(0, 21, n), rng.normal(0, 40, n)
    has_opt, has_optf = rng.random(n) < 0.7, rng.random(n) < 0.6
    nl, nt = rng.integers(0, 4, n), rng.integers(0, 3, n)
    ks = rng.integers(0, 6, (n, K_COLS))
    nw = rng.integers(1, 7, n)
    docs = []
    for i in range(n):
        d = {"body": " ".join(WORDS[int(x)] for x in rng.integers(0, len(WORDS), int(nw[i]))),
             "svc": int(svc[i]), "lat": int(lat[i]), "code": int(code[i]), "latf": float(latf[i]), "t": int(t[i]),
             "ts": int(t[i])}
        if has_opt[i]:
            d["opt"] = int(opt[i])
        if has_optf[i]:
            d["optf"] = float(optf[i])
        if nl[i]:
            d["lvl"] = [int(x) for x in rng.integers(0, 5, int(nl[i]))]
        if nt[i]:
            d["tags"] = [int(x) for x in rng.integers(0, 10, int(nt[i]))]
        for k in range(K_COLS):
            d[f"k{k:02d}"] = int(ks[i, k]) % (k % 5 + 2)
        docs.append(d)
    return docs


def _mapped(ftype: str, v) -> int:
    if ftype == "i64":
        return S.i64_to_u64(int(v))
    if ftype == "f64":
        return S.f64_to_u64(float(v))
    return int(v)


class OptionalColumn(Column):
    """A CARD_OPTIONAL column (at most one value per doc). agg_ref reads a Column with `start` as multi-valued, which
    its exact-sum rule counts against the sum's width; an optional ancestor does not, so it is kept as a doc -> value
    map with `start` None."""

    def __init__(self, ctype: int, per: List[List[int]]):
        super().__init__(ctype, [v[0] for v in per if v])
        self.num_docs = len(per)
        self._by_doc = [v[0] if v else None for v in per]

    def doc_values(self, d: int) -> List[int]:
        v = self._by_doc[d]
        return [] if v is None else [int(v)]

    def empty_docs(self) -> int:
        return self.num_docs - self.num_vals


def _column(docs: List[dict], name: str) -> Column:
    ftype = TYPES[name]
    ctype = {"u64": ffi.COL_U64, "i64": ffi.COL_I64, "f64": ffi.COL_F64}[ftype]
    per = [v if isinstance(v, list) else [v] for v in (d.get(name, []) for d in docs)]
    if all(len(v) == 1 for v in per):
        return Column(ctype, [_mapped(ftype, v[0]) for v in per])
    if all(len(v) <= 1 for v in per):
        return OptionalColumn(ctype, [[_mapped(ftype, x) for x in v] for v in per])
    start = np.concatenate([[0], np.cumsum([len(v) for v in per])]).astype(np.int64)
    return Column(ctype, [_mapped(ftype, x) for v in per for x in v], start)


class WideSplit(Split):
    """A split built from documents, with agg_ref Columns for its fast fields (agg_corpora.Split's node builders)."""

    def __init__(self, split_id: str, docs: List[dict]):
        self.docs = docs
        self.img = S.build_split(docs, MAPPING, split_id)
        self.num_docs = len(docs)
        names = [f["name"] for f in MAPPING["field_mappings"] if f.get("fast") and f["type"] != "datetime"]
        self.by_name: Dict[str, int] = {nm: self.img.column_ord(nm) for nm in names}
        self.cols: Dict[int, Column] = {self.by_name[nm]: _column(docs, nm) for nm in names}


# ---- dense trees of exactly n nodes ----------------------------------------------------------------------------------
CODE_RANGES = [(S.i64_to_u64(-50), S.i64_to_u64(-10)), (S.i64_to_u64(-10), S.i64_to_u64(10)),
               (S.i64_to_u64(0), (1 << 64) - 1)]
TAG_RANGES = [(0, 3), (3, 7), (5, 1 << 40)]


def _bucket(sp: Split, i: int) -> P.Agg:
    return [lambda: sp.terms("svc"), lambda: sp.hist("lat", 500.0), lambda: sp.range("code", CODE_RANGES),
            lambda: sp.terms("lvl"), lambda: sp.hist("optf", 7.5), lambda: sp.terms("opt", missing=0),
            lambda: sp.range("tags", TAG_RANGES), lambda: sp.hist("t", 3600.0, offset=600.0)][i % 8]()


def _metric(sp: Split, i: int) -> P.Agg:
    return sp.stats(("latf", "lat", "opt", "lvl", "code", "optf", "tags")[i % 7])


def count_nodes(aggs) -> int:
    return sum(1 + count_nodes(a.children) for a in aggs)


def depth_of(aggs) -> int:
    return max((1 + depth_of(a.children) for a in aggs), default=0)


def dense_tree(sp: Split, n: int, levels: int) -> List[P.Agg]:
    """n nodes mixing terms, histogram, range and stats over FULL, OPTIONAL and MULTI columns: flat (levels 1),
    bucket > {bucket, stats} (2) or bucket > bucket > stats (3); every tree stays in the dense layout."""
    tops: List[P.Agg] = []
    left, i = n, 0
    while left:
        if levels == 1 or left == 1:
            a = _bucket(sp, i) if i % 3 != 2 else _metric(sp, i)
            left -= 1
        else:
            a = _bucket(sp, i)
            left -= 1
            kids = []
            for j in range(3):
                if not left:
                    break
                if levels == 3 and j == 0 and left >= 3:
                    inner = _bucket(sp, i + j + 1)
                    inner.children = [_metric(sp, i + j), _metric(sp, i + j + 3)]
                    kids.append(inner)
                    left -= 3
                else:
                    kids.append(_metric(sp, i + j) if j % 2 == 0 else _bucket(sp, i + j + 2))
                    left -= 1
            a.children = kids
        tops.append(a)
        i += 1
    assert count_nodes(tops) == n and depth_of(tops) <= levels
    return tops


def fast_plan(sp: Split, n: int) -> List[P.Agg]:
    """n nodes on k_window's fast path: flat terms / histograms over FULL columns with stats children."""
    tops, left, i = [], n, 0
    while left:
        a = [lambda: sp.terms("svc"), lambda: sp.hist("lat", 1000.0), lambda: sp.hist("code", 10.0, offset=5.0),
             lambda: sp.terms(f"k{i % K_COLS:02d}"), lambda: sp.hist("latf", 25.0)][i % 5]()
        left -= 1
        kids = []
        for j in range(min(2, left)):
            kids.append(sp.stats(("lat", "latf", "code", "t")[(i + j) % 4]))
            left -= 1
        a.children = kids
        tops.append(a)
        i += 1
    return tops


def aggscan_flat(sp: Split, n: int) -> List[P.Agg]:
    """n flat terms / histogram nodes over FULL columns of at most 32 bits, without children: what k_aggscan takes
    when n <= QA_MAX_AGGS."""
    return [sp.terms(f"k{i:02d}") if i % 2 else sp.hist("lat", 250.0 * (i + 1)) for i in range(n)]


def aggscan_eligible(aggs, n_cells: int, query_all: bool, max_hits: int, cols_full_le32: bool) -> bool:
    """aggscan_layout's eligibility (engine.cu), restated for one plan: match_all without hits, 1..QA_MAX_AGGS flat
    terms / histogram nodes without `missing` over FULL columns of at most 32 bits, at most QA_MAX_CELLS cells. (The
    engine also needs the plan on the fast path and its columns to fit the two staging slots.)"""
    flat = all(not a.children and a.kind in (ffi.AGG_TERMS, ffi.AGG_HISTOGRAM) and a.missing is None for a in aggs)
    return (query_all and max_hits == 0 and 0 < len(aggs) <= QA_MAX_AGGS and n_cells <= QA_MAX_CELLS and flat and
            cols_full_le32)


# ---- hashed trees ----------------------------------------------------------------------------------------------------
def chain(sp: Split, levels: int, leaf: Optional[P.Agg] = None, ranges: bool = True) -> P.Agg:
    """A chain of `levels` bucket nodes, each the only child of the one before (with `leaf` below the last); without
    `ranges`, terms and histograms only."""
    kinds = [lambda: sp.terms("svc"), lambda: sp.terms("lvl"), lambda: sp.hist("lat", 1250.0),
             lambda: sp.terms("opt", missing=0),
             (lambda: sp.range("code", CODE_RANGES)) if ranges else (lambda: sp.terms("k01")), lambda: sp.terms("tags"),
             lambda: sp.hist("latf", 40.0), lambda: sp.terms("k03")]
    nodes = [kinds[i % len(kinds)]() for i in range(levels)]
    for a, b in zip(nodes, nodes[1:]):
        a.children = [b]
    if leaf is not None:
        nodes[-1].children = [leaf]
    return nodes[0]


def hashed_tree(sp: Split, n: int, levels: int = MAX_LEVELS, leaf: str = "latf") -> List[P.Agg]:
    """A chain of `levels` levels (its deepest node a stats leaf over `leaf`) and siblings up to n nodes."""
    tops = [chain(sp, levels - 1, sp.stats(leaf))]
    i = 0
    while count_nodes(tops) < n:
        if n - count_nodes(tops) >= 2 and i % 2 == 0:
            tops.append(_bucket(sp, i))
            tops[-1].children = [_metric(sp, i)]
        else:
            tops.append(_metric(sp, i) if i % 3 else _bucket(sp, i))
        i += 1
    assert count_nodes(tops) == n and depth_of(tops) == levels
    return tops
