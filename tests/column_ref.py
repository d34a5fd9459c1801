"""A brute-force restatement of fast-field range / exists filters and column sort keys, computed from the arrays the
splits of column_corpora were built from (never from the image).

  * range: a doc matches when ANY of its mapped values lies in [lo, hi], compared in mapped u64 space (so -0.0 sorts
    below 0.0 and NaN above +inf, as the monotonic mapping orders them); exists: the doc has a value;
  * bool: bool_ref's rule (all required clauses, no must_not clause, at least minimum_should_match should clauses,
    else 1 when there is no required clause; the f32 sum of the scored MUST clauses plus that of the matching SHOULD
    clauses);
  * score: a range / exists clause scores its boost, a term 0;
  * order (SegmentPartialHitSortingKey, collector.rs:1082-1118): sort value 1, sort value 2, None last in both
    directions, then the doc id in the direction of the first key; a column's sort value is the doc's first value in
    index order;
  * search_after (collect_top_k_vals, top_k_collector.rs:663-699): a doc is kept when it compares below the
    QwSearchAfter fields, `compare_on_equal` / `precomp_order` breaking the tie of equal sort values.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

from quickwit_b200 import ffi, plan as P, splitgen as S
from column_corpora import Col, Split
import bool_ref

MUST, SHOULD, MUST_NOT, FILTER = ffi.OCCUR_MUST, ffi.OCCUR_SHOULD, ffi.OCCUR_MUST_NOT, ffi.OCCUR_FILTER
ASC, DESC = ffi.ORDER_ASC, ffi.ORDER_DESC


class Q:
    """One query clause, from which both the plan node and the reference are built."""

    def __init__(self, kind: str, occur: int = FILTER, col: Optional[str] = None, lo: int = 0, hi: int = 0,
                 term: Optional[str] = None, children: Sequence["Q"] = (), msm: Optional[int] = None, boost: float = 1.0):
        self.kind, self.occur, self.col, self.lo, self.hi = kind, occur, col, lo, hi
        self.term, self.children, self.msm, self.boost = term, list(children), msm, boost

    def __repr__(self):
        if self.kind == "bool":
            return f"bool[{self.occur}]({', '.join(map(repr, self.children))}; msm={self.msm})"
        if self.kind == "term":
            return f"term[{self.occur}]({self.term})"
        if self.kind == "exists":
            return f"exists[{self.occur}]({self.col})"
        return f"range[{self.occur}]({self.col}, {self.lo:#x}, {self.hi:#x}, boost={self.boost})"


def rng(col: str, lo: int, hi: int, occur: int = FILTER, boost: float = 1.0) -> Q:
    return Q("range", occur, col=col, lo=lo, hi=hi, boost=boost)


def exists(col: str, occur: int = FILTER, boost: float = 1.0) -> Q:
    return Q("exists", occur, col=col, boost=boost)


def term(t: str, occur: int = MUST) -> Q:
    return Q("term", occur, term=t)


def bool_(children: Sequence[Q], msm: Optional[int] = None, occur: int = MUST) -> Q:
    return Q("bool", occur, children=children, msm=msm)


def node(sp: Split, q: Q) -> P.Node:
    if q.kind == "term":
        return P.term(sp.img, "t", q.term, q.occur)
    if q.kind == "range":
        return P.range_(sp.img, q.col, q.lo, q.hi, q.occur, q.boost)
    if q.kind == "exists":
        n = P.exists(sp.img, q.col, q.occur)
        n.boost = q.boost
        return n
    return P.bool_([node(sp, c) for c in q.children], q.msm, q.occur)


def range_mask(c: Col, lo: int, hi: int) -> np.ndarray:
    hit = (c.vals >= np.uint64(lo)) & (c.vals <= np.uint64(hi))
    out = np.zeros(c.num_docs, dtype=bool)
    out[c.doc_of[hit]] = True
    return out


def _leaf(sp: Split, q: Q) -> Tuple[np.ndarray, np.ndarray]:
    """(match mask, f32 score) of a term (unscored), range or exists clause over every doc of the split."""
    n = sp.num_docs
    f32 = np.float32
    if q.kind == "term":
        m = np.zeros(n, dtype=bool)
        m[sp.terms.get(q.term, np.zeros(0, dtype=np.int64))] = True
        return m, np.zeros(n, dtype=f32)
    c = sp.cols.get(q.col)
    if c is None:
        m = np.zeros(n, dtype=bool)
    else:
        m = c.has.copy() if q.kind == "exists" else range_mask(c, q.lo, q.hi)
    return m, np.where(m, f32(q.boost), f32(0)).astype(f32)


def evaluate(sp: Split, q: Q) -> Tuple[np.ndarray, np.ndarray]:
    """(match mask, f32 score) of clause q over every doc of the split (bool_ref's rule over these leaves)."""
    return bool_ref.evaluate(q, lambda x: _leaf(sp, x), sp.num_docs)


class Sort:
    """Up to two (kind, order, column name) keys, as the plan header holds them."""

    def __init__(self, keys: Sequence[Tuple[int, int, Optional[str]]]):
        self.keys = list(keys)

    def spec(self, sp: Split):
        return [(k, o, (sp.ords[c] if c in sp.ords else ffi.ABSENT) if k == ffi.SORT_COLUMN else ffi.ABSENT)
                for k, o, c in self.keys]


def _values(sp: Split, key, score: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """(has, mapped value) of one sort key for every doc."""
    n = sp.num_docs
    if key is None or key[0] in (ffi.SORT_NONE, ffi.SORT_DOCID):
        return np.zeros(n, dtype=bool), np.zeros(n, dtype=np.uint64)
    if key[0] == ffi.SORT_SCORE:
        return np.ones(n, dtype=bool), np.array([S.f64_to_u64(float(x)) for x in score], dtype=np.uint64)
    c = sp.cols.get(key[2])
    if c is None:
        return np.zeros(n, dtype=bool), np.zeros(n, dtype=np.uint64)
    return c.has, np.where(c.has, c.first, np.uint64(0))


def _cmp(order: int, a: np.ndarray, b) -> np.ndarray:
    b = np.uint64(b)
    c = (a > b).astype(np.int64) - (a < b).astype(np.int64)
    return c if order == DESC else -c


def _cmp_opt(order: int, ha: np.ndarray, a: np.ndarray, hb: bool, b: int) -> np.ndarray:
    if hb:
        return np.where(ha, _cmp(order, a, b), -1)    # None sorts after every value
    return np.where(ha, 1, 0)


def top_k(sp: Split, mask: np.ndarray, score: np.ndarray, sort: Sort, K: int,
          sa: Optional[ffi.QwSearchAfter] = None) -> Tuple[int, List[Tuple[int, int, int, int]]]:
    """(num_hits, [(doc, flags, v1, v2)] of the best K docs)."""
    keys = sort.keys + [None] * (2 - len(sort.keys))
    k1, k2 = keys
    if k1 is None or k1[0] == ffi.SORT_NONE:
        k1 = (ffi.SORT_DOCID, DESC, None)
    if k2 is not None and k2[0] == ffi.SORT_DOCID:
        k2 = None   # _doc as the second key extracts None
    o1 = k1[1]
    o2 = k2[1] if k2 is not None else DESC
    h1, v1 = _values(sp, k1, score)
    h2, v2 = _values(sp, k2, score)
    docs = np.arange(sp.num_docs, dtype=np.int64)
    keep = mask.copy()
    if sa is not None and sa.present:
        c = _cmp_opt(o1, h1, v1, bool(sa.has_v1), sa.v1)
        c = np.where(c == 0, _cmp_opt(o2, h2, v2, bool(sa.has_v2), sa.v2), c)
        if sa.compare_on_equal:
            c = np.where(c == 0, sa.precomp_order, c)
            c = np.where(c == 0, _cmp(o1, docs.astype(np.uint64), sa.doc_id), c)
        keep &= c < 0
    idx = np.nonzero(keep)[0]
    # np.lexsort: the last key is the primary one; every key ascending = best first
    def directed(v, order):
        return ~v[idx] if order == DESC else v[idx]
    order = np.lexsort((-idx if o1 == DESC else idx,
                        directed(v2, o2), ~h2[idx],
                        directed(v1, o1), ~h1[idx]))
    best = idx[order[:K]]
    hits = [(int(d), int(h1[d]) | int(h2[d]) << 1, int(v1[d]) if h1[d] else 0, int(v2[d]) if h2[d] else 0) for d in best]
    return int(mask.sum()), hits


def expected(sp: Split, q: Q, sort: Sort, K: int, sa: Optional[ffi.QwSearchAfter] = None):
    mask, score = evaluate(sp, q)
    return top_k(sp, mask, score, sort, K, sa)


def plan(sp: Split, q: Q, sort: Sort, K: int, sa: Optional[ffi.QwSearchAfter] = None, aggs=()) -> bytes:
    return P.make_plan(node(sp, q), K, sort.spec(sp), aggs=aggs, search_after=sa)


def after(hit: Tuple) -> ffi.QwSearchAfter:
    """The QwSearchAfter of paging past `hit` (doc, flags, v1, v2, ...) within its own split."""
    sa = ffi.QwSearchAfter()
    sa.present, sa.has_v1, sa.has_v2 = 1, hit[1] & 1, (hit[1] >> 1) & 1
    sa.v1, sa.v2 = hit[2], hit[3]
    sa.compare_on_equal, sa.precomp_order, sa.doc_id = 1, 0, hit[0]
    return sa


def check(got, sp: Split, q: Q, sort: Sort, K: int, sa=None, scored: bool = False, ctx: str = "", ev=None):
    """`got` (a GPU or oracle result) against the brute force: num_hits and (doc, flags, v1, v2) of every hit, and the
    f32 score bits of a plan ranked by _score (`scored`). `ev(sp, q)` gives (match mask, f32 score); default:
    `evaluate`."""
    mask, score = (ev or evaluate)(sp, q)
    nh, want = top_k(sp, mask, score, sort, K, sa)
    assert got.num_hits == nh, f"{ctx}: num_hits {got.num_hits} != {nh}"
    g = [tuple(int(x) for x in h[:4]) for h in got.hits]
    if g != want:
        for i, (a, b) in enumerate(zip(g, want)):
            if a != b:
                raise AssertionError(f"{ctx}: hit {i} differs: got {a} brute force {b} (n={len(g)}/{len(want)})")
        raise AssertionError(f"{ctx}: hit count {len(g)} != {len(want)}")
    if scored:
        gs = np.array([h[4] for h in got.hits], dtype=np.float32).view(np.uint32)
        ws = score[[h[0] for h in want]].astype(np.float32).view(np.uint32)
        assert np.array_equal(gs, ws), f"{ctx}: f32 score bits differ"


# ---- the cases of the GPU module (the host module runs every one of them on the oracle) --------------------------
U64_MAX = (1 << 64) - 1
SORT_DOC_DESC = Sort([(ffi.SORT_DOCID, DESC, None)])
SORT_DOC_ASC = Sort([(ffi.SORT_DOCID, ASC, None)])


def col_sort(name: str, order: int, second: Optional[Tuple[str, int]] = None) -> Sort:
    keys = [(ffi.SORT_COLUMN, order, name)]
    if second is not None:
        keys.append((ffi.SORT_COLUMN, second[1], second[0]))
    return Sort(keys)


def bounds(c: Col, rs: np.random.Generator) -> List[Tuple[str, int, int]]:
    """(label, lo, hi) at the points where a range test goes wrong: exactly two stored values, one below and one above
    each, between gcd multiples, lo = hi on a stored value and next to it, the column's own min / max, the whole u64
    space, and wholly below or above the column (the compiler's empty shortcut)."""
    if c.num_vals == 0:
        return [("all", 0, U64_MAX)]
    u = np.unique(c.vals)
    a, b = sorted(int(x) for x in u[rs.integers(0, u.size, size=2)])
    dn, up = (lambda x: max(x - 1, 0)), (lambda x: min(x + 1, U64_MAX))
    out = [("stored", a, b), ("inside", up(a), dn(b)), ("outside", dn(a), up(b)), ("lo=hi", a, a),
           ("lo=hi+1", up(a), up(a)), ("lo=hi-1", dn(b), dn(b)), ("min..min", c.min, c.min), ("max..max", c.max, c.max),
           ("all", 0, U64_MAX), ("min..", c.min, U64_MAX), ("..max", 0, c.max)]
    if c.gcd > 1:
        h = c.gcd // 2
        out += [("between gcd", a + h, b + h), ("between gcd lo=hi", a + h, a + h)]
    if c.min > 0:
        out.append(("below", 0, c.min - 1))
    if c.max < U64_MAX:
        out.append(("above", c.max + 1, U64_MAX))
    return out


def filter_columns(sp: Split) -> List[str]:
    return [name for name in sp.cols]


def driver_cases(sp: Split, seed: int = 3):
    """term AND one range / exists filter on every column at every bound point, sorted by that column (or by doc id),
    then term AND 2..4 filters: (label, Q, Sort, K)."""
    rs = np.random.default_rng(seed)
    out = []
    drivers = ("all", "d30", "sparse", "q129")
    for ci, name in enumerate(filter_columns(sp)):
        c = sp.cols[name]
        t = drivers[ci % len(drivers)]
        for bi, (bl, lo, hi) in enumerate(bounds(c, rs)):
            srt = col_sort(name, (ci + bi) % 2) if bi % 3 else SORT_DOC_DESC
            out.append((f"{t} & {name} {bl}", bool_([term(t), rng(name, lo, hi)]), srt, 100))
        out.append((f"{t} & exists {name}", bool_([term(t), exists(name)]), col_sort(name, ASC), 100))
    names = filter_columns(sp)
    for k in range(40):
        nf = 2 + k % 3
        picks = [names[int(i)] for i in rs.choice(len(names), nf, replace=False)]
        fs = []
        for name in picks:
            bl = bounds(sp.cols[name], rs)
            _, lo, hi = bl[int(rs.integers(0, 3))]       # stored / inside / outside: a real fraction of the docs
            fs.append(exists(name) if rs.random() < 0.25 else rng(name, lo, hi))
        out.append((f"d30 & {nf} filters {picks}", bool_([term("d30")] + fs), col_sort(picks[0], k % 2), 1000))
    return out


def _wide(sp: Split, name: str, rs=None) -> Tuple[int, int]:
    """A range over roughly the middle half of a column's values."""
    v = np.sort(sp.cols[name].vals)
    return int(v[v.size // 4]), int(v[3 * v.size // 4])


def scan_cases(sp: Split, seed: int = 4):
    """k_window's scan: a range / exists as the only required clause, as should with minimum_should_match, as
    must_not, nested two and three bool levels deep; scored range clauses under _score."""
    rs = np.random.default_rng(seed)
    out = []
    for name in filter_columns(sp):
        c = sp.cols[name]
        for bl, lo, hi in bounds(c, rs)[:4]:
            out.append((f"only {name} {bl}", bool_([rng(name, lo, hi)]), SORT_DOC_DESC, 100, False))
        out.append((f"only exists {name}", bool_([exists(name)]), SORT_DOC_ASC, 100, False))
    a, b, c3 = "w33", "m53", "o10"
    ra, rb, rc = (rng(x, *_wide(sp, x, rs), occur=SHOULD) for x in (a, b, c3))
    for msm in (None, 1, 2, 3):
        out.append((f"should msm={msm}", bool_([ra, rb, rc], msm), col_sort("w40", DESC), 1000, False))
    out.append(("must_not", bool_([rng("w20", *_wide(sp, "w20", rs)), rng("m9", *_wide(sp, "m9", rs), occur=MUST_NOT),
                                   exists("o63", occur=MUST_NOT)]), col_sort("o33", ASC), 1000, False))
    inner = bool_([rng("m33", *_wide(sp, "m33", rs), occur=SHOULD), exists("o1", occur=SHOULD)], occur=FILTER)
    out.append(("two levels", bool_([rng("w64", *_wide(sp, "w64", rs)), inner]), SORT_DOC_DESC, 4096, False))
    deep = bool_([bool_([rng("g1000", *_wide(sp, "g1000", rs), occur=SHOULD), rng("i64", *_wide(sp, "i64", rs), occur=SHOULD)],
                        occur=SHOULD), exists("o0", occur=MUST_NOT)], occur=FILTER)
    out.append(("three levels", bool_([rng("f64", 0, U64_MAX), bool_([deep, rng("dt", *_wide(sp, "dt", rs))], occur=FILTER)]),
                col_sort("f64", DESC), 1000, False))
    sc = Sort([(ffi.SORT_SCORE, DESC, None)])
    sc_asc = Sort([(ffi.SORT_SCORE, ASC, None)])
    boosts = (0.7, 1.3, 0.1, 2.5)
    must = [rng(x, *_wide(sp, x, rs), occur=MUST, boost=bo) for x, bo in zip(("w33", "m53", "o10", "g3"), boosts)]
    should = [rng(x, *_wide(sp, x, rs), occur=SHOULD, boost=bo) for x, bo in zip(("w12", "m31", "o64", "dt"), boosts)]
    out.append(("scored must", bool_(must[:2]), sc, 1000, True))
    out.append(("scored should", bool_(should), sc, 1000, True))
    out.append(("scored should msm 2", bool_(should, 2), sc_asc, 1000, True))
    out.append(("scored must + should", bool_([must[0], should[0], should[1], must[2]]), sc, 4096, True))
    out.append(("scored exists", bool_([exists("o9", occur=SHOULD, boost=0.3), should[2], exists("m10", occur=SHOULD, boost=3.0)]),
                sc, 1000, True))
    return out


GATHER_TERMS = ("q128", "q129", "sparse", "all")


def gather_cases(sp: Split, seed: int = 5):
    """k_window's candidate gather: term AND range with a second term (the plan stays off k_driver), and two ranges
    (the first scans, the second gathers)."""
    rs = np.random.default_rng(seed)
    out = []
    for t in GATHER_TERMS:
        for name in ("w1", "w33", "w53", "w64", "o11", "m63", "g1000", "f64", "i64"):
            for bl, lo, hi in bounds(sp.cols[name], rs)[:3]:
                out.append((f"{t} & all & {name} {bl}", bool_([term(t), term("all"), rng(name, lo, hi)]), col_sort(name, DESC), 1000))
            out.append((f"{t} & all & exists {name}", bool_([term(t), term("all"), exists(name)]), SORT_DOC_ASC, 1000))
    for x, y in (("w40", "m33"), ("o53", "w9"), ("g3", "m1")):
        out.append((f"{x} then {y}", bool_([rng(x, *_wide(sp, x, rs)), rng(y, *_wide(sp, y, rs))]), col_sort(y, ASC), 1000))
    return out


def sort_cases(sp: Split):
    """Every width and cardinality as the first key, ASC and DESC, K in {1, 10, 1000, 4096}; the key-layout pairs."""
    out = []
    for name in filter_columns(sp):
        for o in (ASC, DESC):
            for K in (1, 10, 1000, 4096):
                out.append((f"{name} {'desc' if o else 'asc'}", name, col_sort(name, o), K))
    return out


def key_pairs(sp: Split) -> List[Tuple[str, str, int]]:
    """(first, second, total key bits) of the pairs whose composite key is exactly 64 bits, exactly 65 bits, and
    three words wide on this split."""
    db = (sp.num_docs - 1).bit_length()
    out = []
    for want in (64, 65):
        b2 = want - db - 2 - 31
        out.append(("w31", f"w{b2}", want))
    out.append(("w64", "w64", db + 130))
    out.append(("w63", "o53", db + 118))
    out.append(("o10", "m11", db + 23))
    for a, b, tb in out:
        assert db + 2 + sp.cols[a].bits + sp.cols[b].bits == tb, (a, b)
    return out
