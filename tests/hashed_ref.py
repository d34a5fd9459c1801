"""The hashed aggregation layout (QwAggEntry, include/qwgpu_format.h) restated from the column values, and the
conversions the tests need between it and the dense layout.

A hashed result is a set of entries, one per (node, parent entry, key) that a matched doc reached. Here an entry is
named by its path: (node, ((ancestor node, key, missing), ...), key, missing), which does not depend on the order in
which the engine handed out entry ids. Keys follow the layout's rules: terms = the raw value (0 and missing = True for
the `missing` bucket), histogram = the bucket index from agg_ref's f64 formula, range = the range index, stats = 0."""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

from quickwit_b200 import ffi, plan as P
from agg_ref import Cell, Column, Sum, _hist_index, _layout, mapped_to_f64, sum_is_exact

NO_PARENT = ffi.AGG_NO_PARENT


def _keys(a: P.Agg, col: Optional[Column], d: int) -> List[Tuple[int, bool]]:
    """(key, missing) of every bucket of node `a` that doc d lands in, once per value that puts it there."""
    vals = col.doc_values(d) if col is not None else []
    if a.kind == ffi.AGG_TERMS:
        if not vals:
            return [(0, True)] if a.missing is not None else []
        return [(col.raw(v), False) for v in vals]
    out = []
    for v in vals:
        if a.kind == ffi.AGG_HISTOGRAM:
            k = _hist_index(a, mapped_to_f64(col.ctype, v))
            if k is not None:
                out.append((k, False))
        else:
            out.extend((r, False) for r, (f, t) in enumerate(a.ranges) if f <= v < t)
    return out


def sparse_cells(aggs: Sequence[P.Agg], cols: Dict[int, Column], docs: Optional[Sequence[int]] = None) -> Dict[tuple, Cell]:
    """{path: Cell} of plan aggregations `aggs` over the matched docs `docs` (None: every doc), the brute force of
    the hashed layout: a dict entry for every (node, parent path, key) some (doc, value path) reaches."""
    lay = _layout(aggs)
    index = {id(a): i for i, (a, _p, _b, _n) in enumerate(lay)}

    def col_of(a):
        return cols.get(a.column) if a.column != ffi.ABSENT else None

    def ancestors(i):
        q, anc = lay[i][1], []
        while q >= 0:
            anc.append(col_of(lay[q][0]))
            q = lay[q][1]
        return anc

    exact = {i: sum_is_exact(col_of(a), ancestors(i)) for i, (a, _p, _b, _n) in enumerate(lay)
             if a.kind == ffi.AGG_STATS and col_of(a) is not None}
    out: Dict[tuple, Cell] = {}

    def visit(a: P.Agg, d: int, path: tuple):
        i = index[id(a)]
        col = col_of(a)
        if a.kind == ffi.AGG_STATS:
            vals = col.doc_values(d) if col is not None else []
            if not vals:
                return
            c = out.setdefault((i, path, 0, False), Cell(Sum(exact[i])))
            for v in vals:
                c.count += 1
                c.min, c.max = min(c.min, v), max(c.max, v)
                c.sum.add(col.raw(v), mapped_to_f64(col.ctype, v))
            return
        for key, missing in _keys(a, col, d):
            c = out.setdefault((i, path, key, missing), Cell())
            c.count += 1
            for ch in a.children:
                visit(ch, d, path + ((i, key, missing),))

    num_docs = max(c.num_docs for c in cols.values())
    for d in (range(num_docs) if docs is None else docs):
        for a in aggs:
            visit(a, int(d), ())
    return out


def entry_paths(entries) -> Dict[tuple, tuple]:
    """{path: cell tuple} of engine entries (node, parent, key, flags, cell); every path must be unique."""
    memo: Dict[int, tuple] = {}

    def path_of(e: int) -> tuple:
        if e not in memo:
            node, parent, key, flags, _cell = entries[e]
            miss = bool(flags & ffi.AGG_ENTRY_MISSING)
            up = () if parent == NO_PARENT else path_of(parent) + ((entries[parent][0], entries[parent][2],
                                                                    bool(entries[parent][3] & ffi.AGG_ENTRY_MISSING)),)
            memo[e] = up
        return memo[e]

    out = {}
    for e, (node, _parent, key, flags, cell) in enumerate(entries):
        k = (node, path_of(e), key, bool(flags & ffi.AGG_ENTRY_MISSING))
        assert k not in out, f"two entries for {k}"
        out[k] = cell
    return out


def assert_entries(entries, want: Dict[tuple, Cell], ctx: str = ""):
    got = entry_paths(entries)
    missing, extra = set(want) - set(got), set(got) - set(want)
    assert not missing and not extra, f"{ctx}: {len(missing)} entries missing (e.g. {sorted(missing)[:3]}), " \
                                      f"{len(extra)} unexpected (e.g. {sorted(extra)[:3]})"
    for k, w in want.items():
        g, c = got[k], f"{ctx}: entry {k}"
        assert g[0] == w.count, f"{c}: count {g[0]} != {w.count}"
        assert (g[2], g[3]) == (w.min, w.max), f"{c}: min/max {(g[2], g[3])} != {(w.min, w.max)}"
        if w.sum is None:
            assert g[1] == 0, f"{c}: sum_bits {g[1]} of a bucket cell"
        else:
            w.sum.check(g[1], c)


def dense_to_entries(aggs: Sequence[P.Agg], cells) -> List[tuple]:
    """Engine-style entries (node, parent, key, flags, cell) of a dense cell list (the oracle's): one entry per bucket
    cell with a doc count and per stats cell with a value, parents before children."""
    lay = _layout(aggs)
    entries: List[tuple] = []

    def walk(i: int, parent_entry: int, parent_cell: int):
        a, _p, base, _n = lay[i]
        children = [j for j, (_a, p, _b, _m) in enumerate(lay) if p == i]
        if a.kind == ffi.AGG_STATS:
            c = cells[base + parent_cell]
            if c[0]:
                entries.append((i, parent_entry, 0, 0, tuple(c)))
            return
        for k in range(a.num_buckets):
            cell = parent_cell * a.num_buckets + k
            c = cells[base + cell]
            if not c[0]:
                continue
            miss = a.kind == ffi.AGG_TERMS and a.missing is not None and k == a.num_buckets - 1
            entries.append((i, parent_entry, 0 if miss else k, ffi.AGG_ENTRY_MISSING if miss else 0, tuple(c)))
            me = len(entries) - 1
            for j in children:
                walk(j, me, cell)

    for i, (_a, p, _b, _n) in enumerate(lay):
        if p < 0:
            walk(i, NO_PARENT, 0)
    return entries


def entries_to_dense(aggs: Sequence[P.Agg], entries) -> List[tuple]:
    """The dense cell list of engine entries (plans whose dense layout is small enough to hold)."""
    lay = _layout(aggs)
    total = sum(n for *_x, n in lay)
    out = [(0, 0, (1 << 64) - 1, 0)] * total
    cell_of: Dict[int, int] = {}

    def cell(e: int) -> int:
        if e not in cell_of:
            node, parent, key, _flags, _c = entries[e]
            a = lay[node][0]
            pc = 0 if parent == NO_PARENT else cell(parent)
            cell_of[e] = pc if a.kind == ffi.AGG_STATS else pc * a.num_buckets + (
                a.num_buckets - 1 if entries[e][3] & ffi.AGG_ENTRY_MISSING else key)
        return cell_of[e]

    for e, (node, _parent, _key, _flags, c) in enumerate(entries):
        out[lay[node][2] + cell(e)] = tuple(c)
    return out
