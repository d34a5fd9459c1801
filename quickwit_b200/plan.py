"""Seam-C plan construction (include/qwgpu_format.h QwPlanHeader/QwPlanNode/QwAggNode) from Python.

The C++ host compiles plans from `SearchRequest` protobuf + QueryAst JSON (`qwgpu_compile_plan`);
these helpers build the same bytes by hand, which is what the plan-level parity tests use.
"""
from __future__ import annotations

import ctypes as C
import struct
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import ffi
from .splitgen import SplitImage



def bm25_weight(doc_freq: int, num_docs: int, boost: float = 1.0) -> float:
    """tantivy Bm25Weight: idf * (1 + K1) * boost in f32 (SURVEY.md Appendix A.3) — computed by the
    C++ host (`qwgpu_bm25_weight`) so hand-built plans carry the exact weights compiled plans do."""
    return float(ffi.img_lib().qwgpu_bm25_weight(doc_freq, num_docs, boost))


class Node:
    def __init__(self, kind, occur=ffi.OCCUR_MUST, boost=1.0, children: Sequence["Node"] = (),
                 min_should_match: Optional[int] = None, term_ord=ffi.ABSENT, field_id=0,
                 weight=0.0, column=ffi.ABSENT, lo=0, hi=0):
        self.kind, self.occur, self.boost, self.children = kind, occur, boost, list(children)
        self.msm, self.term_ord, self.field_id, self.weight = min_should_match, term_ord, field_id, weight
        self.column, self.lo, self.hi = column, lo, hi


def term(img: SplitImage, field: str, text: str, occur=ffi.OCCUR_MUST, boost: float = 1.0) -> Node:
    t = img.term_ord(field, text)
    if t < 0:
        return Node(ffi.NODE_TERM, occur)
    return Node(ffi.NODE_TERM, occur, boost, term_ord=t, weight=bm25_weight(img.doc_freq(t), img.num_docs, boost))


def phrase(img: SplitImage, field: str, terms: Sequence[str], occur=ffi.OCCUR_MUST, boost: float = 1.0) -> Node:
    """tantivy PhraseQuery (slop 0) over `terms` in order; any term absent from the split -> matches nothing."""
    ords = [img.term_ord(field, t) for t in terms]
    if any(o < 0 for o in ords) or len(ords) < 2:
        return Node(ffi.NODE_NONE, occur)
    dfs = (C.c_uint64 * len(ords))(*[img.doc_freq(o) for o in ords])
    w = float(ffi.img_lib().qwgpu_bm25_phrase_weight(dfs, len(ords), img.num_docs, boost))
    kids = [Node(ffi.NODE_TERM, ffi.OCCUR_MUST, 1.0, term_ord=o, field_id=img.field_names().index(field), weight=bm25_weight(img.doc_freq(o), img.num_docs), lo=k)
            for k, o in enumerate(ords)]
    return Node(ffi.NODE_PHRASE, occur, boost, children=kids, field_id=img.field_names().index(field), weight=w)


def prefix_expansions(img: SplitImage, field: str, prefix: bytes | str, max_expansions: int) -> List[int]:
    """Term ords of the field's first `max_expansions` terms, in byte order, that start with `prefix` (the
    expansion of a phrase prefix in one split)."""
    if isinstance(prefix, str):
        prefix = prefix.encode()
    names = img.field_names()
    if field not in names:
        return []
    _h, _s, tbytes, fields, terms, _c = img._directory()
    f = fields[names.index(field)]
    out: List[int] = []
    for t in range(f.first_term, f.first_term + f.num_terms):
        if len(out) >= max_expansions:
            break
        b = tbytes[terms[t].bytes_off: terms[t].bytes_off + terms[t].bytes_len]
        if b.startswith(prefix):
            out.append(t)
        elif b > prefix:
            break
    return out


def phrase_prefix(img: SplitImage, field: str, tokens: Sequence[str], max_expansions: int = 50,
                  occur=ffi.OCCUR_MUST, boost: float = 1.0) -> Node:
    """tantivy PhrasePrefixQuery over `tokens` (the last one is the prefix), never scored. One token: the unscored
    set filter of its expansions; more: a PHRASE_PREFIX node. An absent exact term or no expansion matches nothing."""
    fid = img.field_names().index(field) if field in img.field_names() else 0
    ords = [img.term_ord(field, t) for t in tokens[:-1]]
    exps = prefix_expansions(img, field, tokens[-1], max_expansions)
    if any(o < 0 for o in ords) or not exps:
        return Node(ffi.NODE_NONE, occur)

    def kid(o, lo, occ=ffi.OCCUR_MUST):
        return Node(ffi.NODE_TERM, occ, 1.0, term_ord=o, field_id=fid, weight=bm25_weight(img.doc_freq(o), img.num_docs), lo=lo)

    if not ords:
        inner = Node(ffi.NODE_BOOL, ffi.OCCUR_FILTER, children=[kid(o, 0, ffi.OCCUR_SHOULD) for o in exps])
        return Node(ffi.NODE_BOOL, occur, children=[inner])
    k = len(ords)
    kids = [kid(o, i) for i, o in enumerate(ords)] + [kid(o, k) for o in exps]
    return Node(ffi.NODE_PHRASE_PREFIX, occur, boost, children=kids, field_id=fid, lo=k)


def phrase_prefix_as_phrases(node: Node, occur: Optional[int] = None) -> Node:
    """The same match set as a multi-token PHRASE_PREFIX node, as a bool that ORs one plain phrase per expansion
    (scores aside: the phrases are scored where they sit in a scoring clause, the phrase prefix never is)."""
    assert node.kind == ffi.NODE_PHRASE_PREFIX
    k = node.lo
    exact, exps = node.children[:k], node.children[k:]
    phrases = [Node(ffi.NODE_PHRASE, ffi.OCCUR_SHOULD, 1.0, children=list(exact) + [e], field_id=node.field_id) for e in exps]
    return Node(ffi.NODE_BOOL, node.occur if occur is None else occur, children=phrases)


def term_set(img: SplitImage, field: str, ords: Sequence[int], occur=ffi.OCCUR_FILTER) -> Node:
    """A TERM_SET node (the expansions of a regex query): a doc matches when it holds any of the term ords `ords` of
    `field` (ascending). Never scored. No ords: matches nothing."""
    if not ords:
        return Node(ffi.NODE_NONE, occur)
    fid = img.field_names().index(field)
    kids = [Node(ffi.NODE_TERM, ffi.OCCUR_SHOULD, term_ord=o, field_id=fid, weight=bm25_weight(img.doc_freq(o), img.num_docs))
            for o in ords]
    return Node(ffi.NODE_TERM_SET, occur, children=kids, field_id=fid)


def col_set(img: SplitImage, column: str, values: Sequence[int], occur=ffi.OCCUR_FILTER) -> Node:
    """A COL_SET node: a doc matches when one of its values in `column` equals one of `values` (mapped-u64 space;
    sorted and deduplicated here). Never scored. No values: matches nothing."""
    vals = sorted(set(values))
    if not vals:
        return Node(ffi.NODE_NONE, occur)
    c = img.column_ord(column)
    c = c if c >= 0 else ffi.ABSENT
    kids = [Node(ffi.NODE_RANGE, ffi.OCCUR_SHOULD, column=c, lo=v, hi=v) for v in vals]
    return Node(ffi.NODE_COL_SET, occur, children=kids, column=c)


def range_(img: SplitImage, column: str, lo: int, hi: int, occur=ffi.OCCUR_FILTER, boost=1.0) -> Node:
    c = img.column_ord(column)
    return Node(ffi.NODE_RANGE, occur, boost, column=c if c >= 0 else ffi.ABSENT, lo=lo, hi=hi)


def exists(img: SplitImage, column: str, occur=ffi.OCCUR_MUST) -> Node:
    c = img.column_ord(column)
    return Node(ffi.NODE_EXISTS, occur, column=c if c >= 0 else ffi.ABSENT)


def match_all(occur=ffi.OCCUR_MUST) -> Node:
    return Node(ffi.NODE_ALL, occur)


def bool_(children: Sequence[Node], min_should_match: Optional[int] = None, occur=ffi.OCCUR_MUST) -> Node:
    return Node(ffi.NODE_BOOL, occur, children=children, min_should_match=min_should_match)


def cache(node: Node, occur: Optional[int] = None) -> Node:
    """A CACHE node over `node` (the reference's CacheNode): the same docs, read from the context's predicate cache when
    it is enabled. Never scored. `occur` defaults to the node's own; the child takes MUST."""
    child = Node(node.kind, ffi.OCCUR_MUST, node.boost, children=node.children, min_should_match=node.msm,
                 term_ord=node.term_ord, field_id=node.field_id, weight=node.weight, column=node.column, lo=node.lo, hi=node.hi)
    return Node(ffi.NODE_CACHE, node.occur if occur is None else occur, children=[child])


def _flatten(root: Node) -> List[ffi.QwPlanNode]:
    out: List[ffi.QwPlanNode] = []
    queue: List[Tuple[Node, int]] = []

    def emit(n: Node) -> int:
        idx = len(out)
        pn = ffi.QwPlanNode()
        pn.kind, pn.occur, pn.boost = n.kind, n.occur, n.boost
        pn.min_should_match = ffi.ABSENT if n.msm is None else n.msm
        pn.term_ord, pn.field_id, pn.bm25_weight = n.term_ord, n.field_id, n.weight
        pn.column, pn.lo, pn.hi = n.column, n.lo, n.hi
        out.append(pn)
        return idx

    emit(root)
    queue.append((root, 0))
    while queue:
        n, idx = queue.pop(0)
        if n.children:
            out[idx].first_child = len(out)
            out[idx].num_children = len(n.children)
            kids = [(c, emit(c)) for c in n.children]
            queue.extend(kids)
    return out


class Agg:
    def __init__(self, kind, column=ffi.ABSENT, num_buckets=1, children: Sequence["Agg"] = (), interval=0.0,
                 offset=0.0, base_pos=0, bounds: Optional[Tuple[float, float]] = None,
                 ranges: Sequence[Tuple[int, int]] = (), missing: Optional[int] = None):
        self.kind, self.column, self.num_buckets, self.children = kind, column, num_buckets, list(children)
        self.interval, self.offset, self.base_pos, self.bounds = interval, offset, base_pos, bounds
        self.ranges, self.missing = list(ranges), missing
        # composite source (see composite()): QW_AGG_COMP_* flags, the split's `after` bound, the page size
        self.comp, self.comp_after, self.comp_size = 0, 0, 0


def composite(sources: Sequence[Agg], size: int, children: Sequence[Agg] = (), desc: Sequence[int] = (),
              after: Optional[Sequence[Tuple[int, int]]] = None) -> Agg:
    """A composite aggregation as the plan holds it: `sources` (TERMS / HISTOGRAM nodes, `missing` set for a
    missing_bucket source) chained, each the only child of the one before, `children` below the last. `desc`: indices
    of the descending sources. `after`: per source (bound, QW_AGG_COMP_* after flags) in the node's key space, as
    the lowering resolves it for a split. Returns the first source."""
    for i, s in enumerate(sources):
        last = i == len(sources) - 1
        s.comp = ffi.AGG_COMP_LEVEL | (ffi.AGG_COMP_LAST if last else 0) | (ffi.AGG_COMP_DESC if i in desc else 0) | \
            (ffi.AGG_COMP_MISSING if s.missing is not None else 0)
        if after is not None:
            s.comp_after = after[i][0]
            s.comp |= ffi.AGG_COMP_HAS_AFTER | after[i][1]
        s.comp_size = size
        s.children = list(children) if last else [sources[i + 1]]
    return sources[0]


def _f64_bits(missing: Optional[float]) -> Optional[int]:
    return None if missing is None else struct.unpack("<Q", struct.pack("<d", float(missing)))[0]


def percentiles(column: int, num_bins: int, missing: Optional[float] = None) -> Agg:
    """A percentiles node over `column`: `num_bins` = the bins of the split's boundary table for that column (the
    engine builds the table and refuses another count), `missing` = the value of docs without one (kept as f64 bits)."""
    return Agg(ffi.AGG_PERCENTILES, column=column, num_buckets=num_bins + (missing is not None), missing=_f64_bits(missing))


def stats(column: int, missing: Optional[float] = None) -> Agg:
    """A stats node (stats / avg / sum / min / max / value_count) over `column`, ffi.ABSENT when the split lacks it;
    `missing` = the value of docs without one (kept as f64 bits: the device only counts those docs)."""
    return Agg(ffi.AGG_STATS, column=column, missing=_f64_bits(missing))


def _flatten_aggs(tops: Sequence[Agg]) -> List[ffi.QwAggNode]:
    out: List[ffi.QwAggNode] = []

    def emit(a: Agg, parent: int) -> int:
        idx = len(out)
        g = ffi.QwAggNode()
        g.kind, g.parent, g.column, g.num_buckets = a.kind, parent, a.column, a.num_buckets
        g.interval, g.offset, g.base_pos = a.interval, a.offset, a.base_pos
        if a.bounds is not None:
            g.has_bounds, g.bound_min, g.bound_max = 1, a.bounds[0], a.bounds[1]
        g.num_ranges = len(a.ranges)
        for i, (f, t) in enumerate(a.ranges):
            g.range_from[i], g.range_to[i] = f, t
        if a.missing is not None:
            g.has_missing, g.missing_value = 1, a.missing
        if a.comp:
            g.reserved, g.range_from[0], g.range_to[0] = a.comp, a.comp_after, a.comp_size
        out.append(g)
        return idx

    pending: List[Tuple[Agg, int]] = [(a, emit(a, ffi.ABSENT)) for a in tops]
    while pending:
        a, idx = pending.pop(0)
        if a.children:
            out[idx].first_child = len(out)
            out[idx].num_children = len(a.children)
            pending.extend([(c, emit(c, idx)) for c in a.children])
    return out


def make_plan(root: Node, max_hits: int, sort: Sequence[Tuple[int, int, int]] = ((ffi.SORT_DOCID, ffi.ORDER_DESC, ffi.ABSENT),),
              aggs: Sequence[Agg] = (), search_after: Optional[ffi.QwSearchAfter] = None) -> bytes:
    """sort: up to two (kind, order, column) triples. Returns the plan blob."""
    nodes = _flatten(root)
    agg_nodes = _flatten_aggs(aggs)
    h = ffi.QwPlanHeader()
    h.magic, h.version = ffi.PLAN_MAGIC, 1
    h.num_nodes, h.num_aggs, h.max_hits = len(nodes), len(agg_nodes), max_hits
    h.scoring = int(any(k == ffi.SORT_SCORE for k, _, _ in sort))
    h.count_only = int(max_hits == 0 and not agg_nodes)
    for i, (k, o, c) in enumerate(sort[:2]):
        h.sort[i].kind, h.sort[i].order, h.sort[i].column = k, o, c
    if len(sort) < 2:
        h.sort[1].kind, h.sort[1].order, h.sort[1].column = ffi.SORT_NONE, ffi.ORDER_DESC, ffi.ABSENT
    if search_after is not None:
        h.search_after = search_after
    return bytes(h) + b"".join(bytes(n) for n in nodes) + b"".join(bytes(a) for a in agg_nodes)
