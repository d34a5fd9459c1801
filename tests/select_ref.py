"""k_select's composite keys and its unsampled selection path, restated from the source arrays, and the cases that drive
each step of it to an edge (kernels.cuh k_select, select_cut, pick_digit; device_types.h DKeySpec).

Two restatements, both in plain Python integers:
  * `Layout.keys`: every matched doc's 192-bit composite key, [has1][r1:rbits0] [has2][r2:rbits1] [doc':doc_bits] left
    aligned, built from the column values (raw = (v - min) / gcd, r = raw for DESC and raw_max - raw for ASC, 0 without
    a value) or the f32 score (a 10-bit linear bucket, then the order-preserving f32 bits). Sorting the keys gives the
    expected hits; `lexsort_docs` orders the same docs from the values alone, None last, as an independent check.
  * `restate`: what the exact (unsampled) path does with those keys: the candidate set that the radix select of
    pick_digit leaves (sampled == 0, 11-bit digits level by level, done once the candidates fit qw_cand_cap(K)), then on
    those candidates select_cut's stop shift and threshold, the survivor count m, the branch (rank, or sort_all_block
    above QW_SEL_MAX survivors) and the bucket position `at`. It only labels a case; the expected hits always come from
    the sorted keys.

A case is one split with the docs its plan matches. Docs that only pin a column's range (values 0, 1 and 2^64 - 1:
min 0, gcd 1, 64 bits) are left out of the match set by a term `m` (k_driver) and a selector column `sel` (k_window), so
that every column key is 64 bits wide and the matched docs can be placed anywhere in it, in both directions."""
from __future__ import annotations

import random
from collections import Counter
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from quickwit_b200 import ffi, plan as P, splitgen as S
from column_corpora import Col
from helpers import bm25_contributions, bm25_norm
from score_edges_ref import lin as score_lin, score_scale

KEY_BITS = 192
DIGIT_BITS = 11          # QW_DIGIT_BITS
CAND_CAP = 8192          # QW_CAND_CAP
MAX_TOPK = 4096          # QW_MAX_TOPK
SEL_MAX = 2048           # QW_SEL_MAX
RANK_BITS = 10           # QW_RANK_BITS
U64 = (1 << 64) - 1
DESC, ASC = ffi.ORDER_DESC, ffi.ORDER_ASC


def cand_cap(K: int) -> int:
    """qw_cand_cap"""
    return CAND_CAP if K <= MAX_TOPK else (2 * K + 1023) & ~1023


def f32_ordered(s) -> int:
    b = int(np.float32(s).view(np.uint32))
    return (~b & 0xFFFFFFFF) if b & 0x80000000 else (b | 0x80000000)


# ---- the key ---------------------------------------------------------------------------------------------------------
class Layout:
    """The key of one plan on one split. fields: up to two of ("col", order, Col), ("score", order, None), and
    ("doc", order, None) for a doc-id first key (no bits). `scores` (f32 per doc) and `scale` for `_score` fields."""

    def __init__(self, num_docs: int, fields: Sequence[Tuple[str, int, Optional[Col]]], scores=None, scale=None):
        self.num_docs, self.fields, self.scores, self.scale = num_docs, list(fields), scores, scale
        self.doc_bits = (num_docs - 1).bit_length() if num_docs else 0
        self.desc1 = self.fields[0][1] == DESC
        self.widths = []  # (hasbit, rbits) per field
        for i, (kind, order, col) in enumerate(self.fields):
            if kind == "col":
                self.widths.append((1, col.bits))
            elif kind == "score":
                self.widths.append((1, 42 if i == 0 else 32))
            else:
                self.widths.append((0, 0))
        self.total_bits = self.doc_bits + sum(h + r for h, r in self.widths)
        if self.fields[0][0] == "score":
            self.lin = score_lin(np.asarray(scores, dtype=np.float32), scale, self.desc1)

    def key(self, d: int) -> int:
        k = 0
        for i, ((kind, order, col), (hb, rb)) in enumerate(zip(self.fields, self.widths)):
            desc = order == DESC
            if kind == "col":
                has = bool(col.has[d])
                r = 0
                if has:
                    raw = (int(col.first[d]) - col.min) // col.gcd
                    r = raw if desc else ((1 << rb) - 1) - raw
                k = (k << 1 | int(has)) << rb | r
            elif kind == "score":
                s = self.scores[d]
                o = f32_ordered(s)
                r = o if desc else (~o & 0xFFFFFFFF)
                if i == 0:
                    r |= int(self.lin[d]) << 32
                k = (k << 1 | 1) << rb | r
        docr = d if self.desc1 else ((1 << self.doc_bits) - 1) - d
        k = k << self.doc_bits | docr
        return k << (KEY_BITS - self.total_bits)

    def keys(self, docs) -> List[int]:
        return [self.key(int(d)) for d in docs]

    def brute_docs(self, docs) -> List[int]:
        """The matched docs best first: the keys sorted, decoded back to the doc id."""
        mask = (1 << self.doc_bits) - 1
        out = []
        for k in sorted(self.keys(docs), reverse=True):
            docr = (k >> (KEY_BITS - self.total_bits)) & mask
            out.append(docr if self.desc1 else mask - docr)
        return out

    def lexsort_docs(self, docs) -> List[int]:
        """The same order from the values alone (numpy lexsort; None last in both directions, doc id last in the first
        key's direction): SegmentPartialHitSortingKey, independent of the key layout."""
        d = np.asarray(docs, dtype=np.int64)
        cols = [-d if self.desc1 else d]
        for kind, order, col in reversed(self.fields):
            if kind == "col":
                v = col.first[d].astype(np.uint64)
                cols.append(~v if order == DESC else v)
                cols.append(~col.has[d])  # False (has a value) first
            elif kind == "score":
                s = np.asarray(self.scores, dtype=np.float32)[d].astype(np.float64)
                cols.append(-s if order == DESC else s)
        return [int(x) for x in d[np.lexsort(tuple(cols))]]


# ---- the unsampled selection path -------------------------------------------------------------------------------------
def _digit(k: int, level: int) -> int:
    """key_digit: 11-bit digit `level` from the key's most significant bit (zeros past bit 192)"""
    return ((k << DIGIT_BITS) >> (KEY_BITS + DIGIT_BITS - DIGIT_BITS * (level + 1))) & 2047


def radix_candidates(keys: Sequence[int], K: int, total_bits: int) -> Tuple[List[int], int]:
    """pick_digit with sampled == 0, level by level, then the collect pass (candidates: key >= threshold).
    Returns the candidates and the number of histogram levels."""
    cap = cand_cap(K)
    tkey, prefix_bits, above, level = 0, 0, 0, 0
    while True:
        if level == 0:
            ranked = keys
        else:
            sh = KEY_BITS - prefix_bits
            ranked = [k for k in keys if k >> sh == tkey >> sh]
        hist = Counter(_digit(k, level) for k in ranked)
        base_above = 0 if level == 0 else above
        target = K - base_above if K > base_above else 1
        run, sel = 0, None
        for t in range(2047, -1, -1):
            before, run = run, run + hist.get(t, 0)
            if before < target <= run:
                sel = (t, before)
                break
        if sel is None:  # fewer than `target` ranked docs: keep everything matching the current prefix
            if level == 0:
                tkey, prefix_bits = 0, 0
            level += 1
            break
        o = level * DIGIT_BITS
        if level == 0:
            tkey = 0
        sh = KEY_BITS - o - DIGIT_BITS
        tkey |= sel[0] << sh if sh >= 0 else sel[0] >> -sh
        prefix_bits = o + DIGIT_BITS
        above = base_above + sel[1]
        done = above + hist[sel[0]] <= cap
        level += 1
        if done or level * DIGIT_BITS >= total_bits:
            break
    return [k for k in keys if k >= tkey], level


def select_cut(w0: Sequence[int], K: int) -> Tuple[int, Optional[int]]:
    """select_cut over the candidates' first key words: (threshold word, the last shift it resolved; None when every
    candidate survives without a cut)."""
    n = len(w0)
    if n <= K:
        return 0, None
    cap = SEL_MAX
    while cap < K:
        cap <<= 1
    prefix, need, stop = 0, K, None
    for shift in range(56, -1, -8):
        himask = 0 if shift == 56 else (U64 << (shift + 8)) & U64
        hist = Counter((v >> shift) & 255 for v in w0 if (v & himask) == prefix)
        run = 0
        for b in range(255, -1, -1):
            before, run = run, run + hist.get(b, 0)
            if before < need <= run:
                break
        prefix |= b << shift
        need -= before
        stop = shift
        if (K - need) + hist[b] <= cap:
            break
    return prefix, stop


class Label:
    """What the unsampled path does with one split: candidates n, radix levels, cut stop shift, survivors m, branch,
    and (rank branch) the bits every survivor shares and the bucket position."""

    def __init__(self, keys: Sequence[int], K: int, total_bits: int):
        cands, self.levels = radix_candidates(keys, K, total_bits)
        self.n = len(cands)
        w0 = [k >> 128 for k in cands]
        self.thr, self.stop = select_cut(w0, K)
        surv = [k for k, w in zip(cands, w0) if w >= self.thr]
        self.m = len(surv)
        self.branch = "rank" if self.m <= SEL_MAX else "sort"
        self.common = self.at = None
        if self.branch == "rank" and self.m:
            x = 0
            for k in surv:
                x |= k ^ surv[0]
            self.common = KEY_BITS - x.bit_length()
            self.at = min(self.common, KEY_BITS - RANK_BITS)
        self.zero_key = 0 in cands

    def __repr__(self):
        return (f"n={self.n} levels={self.levels} stop={self.stop} m={self.m} branch={self.branch} "
                f"common={self.common} at={self.at}")


def restate(keys: Sequence[int], K: int, total_bits: int) -> Label:
    return Label(keys, K, total_bits)


# ---- cases -----------------------------------------------------------------------------------------------------------
class Case:
    """One split and one plan: `vals[name]` = (mapped values, has) per doc for the u64 columns a and b, `matched` the
    docs the plan matches, `sort` [(kind, order, column name or None)], K. `target`: what the case was built to reach
    (keys of Label, checked on the host)."""

    def __init__(self, name, num_docs, matched, vals, sort, K, target=None):
        self.name, self.num_docs, self.K = name, num_docs, K
        self.matched = np.asarray(sorted(matched), dtype=np.int64)
        self.vals, self.sort, self.target = vals, sort, dict(target or {})
        self.cols: Dict[str, Col] = {}
        for cname, (v, has) in vals.items():
            v = np.asarray(v, dtype=np.uint64)
            has = np.asarray(has, dtype=bool)
            if has.all():
                self.cols[cname] = Col(ffi.COL_U64, ffi.CARD_FULL, v, num_docs)
            else:
                docs = np.flatnonzero(has)
                self.cols[cname] = Col(ffi.COL_U64, ffi.CARD_OPTIONAL, v[docs], num_docs, docs=docs)
        sel = np.zeros(num_docs, dtype=np.uint64)
        sel[self.matched] = 1
        self.cols["sel"] = Col(ffi.COL_U64, ffi.CARD_FULL, sel, num_docs)
        self._label = None

    def layout(self) -> Layout:
        f = [(kind, order, self.cols[c] if kind == "col" else None) for kind, order, c in self.sort]
        return Layout(self.num_docs, f)

    def label(self) -> Label:
        if self._label is None:
            lay = self.layout()
            self._label = restate(lay.keys(self.matched), self.K, lay.total_bits)
        return self._label

    def image(self, split_id: str):
        b = S._Builder(self.num_docs)
        fid = b.add_field("t", 0, ffi.TOK_RAW, None, len(self.matched))
        b.add_term(fid, b"m", self.matched.astype(np.uint32), None)
        for cname in sorted(self.cols):
            c = self.cols[cname]
            b.add_column(cname, c.ctype, c.card, c.vals, c.index())
        return b.finish(split_id)

    def plan(self, img, route: str, K: Optional[int] = None) -> bytes:
        sel = P.range_(img, "sel", 1, 1, occur=ffi.OCCUR_FILTER)
        if route == "driver":
            root = P.bool_([P.term(img, "t", "m", occur=ffi.OCCUR_MUST), sel])
        else:
            root = P.bool_([sel])
        sort = []
        for kind, order, c in self.sort:
            if kind == "col":
                sort.append((ffi.SORT_COLUMN, order, img.column_ord(c)))
            else:
                sort.append((ffi.SORT_DOCID, order, ffi.ABSENT))
        return P.make_plan(root, self.K if K is None else K, sort)


def _filled(n, fillers, rest):
    """values of one column: the range-pinning values on the filler docs, `rest` (doc -> value) elsewhere"""
    v = [0] * n
    for d, x in zip(fillers, (0, 1, U64)):
        v[d] = x
    for d, x in rest.items():
        v[d] = x
    return v


def _value(r: int, order: int) -> int:
    """the u64 value whose rank in a 64-bit column (min 0, gcd 1) is r"""
    return r if order == DESC else U64 - r


def _two_col_case(name, n, fillers, matched, key130, orders, K, target):
    """matched doc d gets the 130 value bits key130[d] = [has_a][r_a:64][has_b][r_b:64] (r = 0 without a value)."""
    va, vb = {}, {}
    ha = [True] * n
    hb = [True] * n
    for d in matched:
        k = key130[d]
        has_a, r_a = k >> 129 & 1, k >> 65 & U64
        has_b, r_b = k >> 64 & 1, k & U64
        assert (has_a or not r_a) and (has_b or not r_b)
        ha[d], hb[d] = bool(has_a), bool(has_b)
        va[d] = _value(r_a, orders[0]) if has_a else 0
        vb[d] = _value(r_b, orders[1]) if has_b else 0
    vals = {"a": (_filled(n, fillers, va), ha), "b": (_filled(n, fillers, vb), hb)}
    return Case(name, n, matched, vals, [("col", orders[0], "a"), ("col", orders[1], "b")], K, target)


AT_VALUE_TARGETS = [0, 1, 2, 9] + list(range(53, 67)) + list(range(117, 130))
AT_DOC_TARGETS = [(130, 0), (131, 1), (135, 5), (140, 10)]  # (p, doc' bits shared), doc_bits 11


def at_cases(orders) -> List[Case]:
    """Survivors sharing exactly p leading key bits: two 64-bit columns, K <= 2048 and at most 2048 matched docs (the
    rank path). p < 130: the value bits below p are random, bit p takes both values (the has bits are 1 except at p);
    p >= 130: every matched doc ties on both columns, and their doc' fill one aligned block of 2^(11 - j) (j = p - 130)."""
    out = []
    tag = f"{'d' if orders[0] == DESC else 'a'}{'d' if orders[1] == DESC else 'a'}"
    for p in AT_VALUE_TARGETS:
        rng = random.Random(1000 + p + 7 * orders[0])
        n, fillers = 1603, (0, 1, 2)
        matched = list(range(3, n))
        base = rng.getrandbits(130) | 1 << 129 | 1 << 64
        key130 = {}
        for i, d in enumerate(matched):
            k = (base >> (130 - p) << (130 - p)) if p else 0
            k |= (i & 1 if i < 2 else rng.getrandbits(1)) << (129 - p)
            k |= rng.getrandbits(129 - p)
            if p != 0:
                k |= 1 << 129
            if p != 65:
                k |= 1 << 64 if p < 65 else (base & 1 << 64)
            if not k >> 129 & 1:
                k &= ~(U64 << 65)
            if not k >> 64 & 1:
                k &= ~U64
            key130[d] = k
        K = 2048 if p < DIGIT_BITS else (777 if p % 2 else 1600)
        out.append(_two_col_case(f"at{p}-{tag}", n, fillers, matched, key130, orders, K, {"branch": "rank", "common": p}))
    for p, j in AT_DOC_TARGETS:
        rng = random.Random(2000 + p + 7 * orders[0])
        n, D = 2048, 11
        fillers = (0, 1, 2)
        size = 1 << (D - j)
        start = 0 if j == 0 else (1024 if j == 1 else 512)
        docs = [dr if orders[0] == DESC else (1 << D) - 1 - dr for dr in range(start, start + size)]
        matched = sorted(d for d in docs if d not in fillers)
        base = rng.getrandbits(130) | 1 << 129 | 1 << 64
        key130 = {d: base for d in matched}
        K = min(len(matched), 1500) if j < 2 else 2048
        out.append(_two_col_case(f"at{p}-{tag}", n, fillers, matched, key130, orders, K, {"branch": "rank", "common": p}))
    return out


CUT_SHIFTS = [56, 48, 40, 32, 24, 16, 8, 0]


def cut_cases() -> List[Case]:
    """select_cut stopping at each shift. One 64-bit column a, first word w0 = [1][r_a >> 1]. For shift s <= 48, 8192
    matched docs share the w0 bits above s + 8 (and so the level-0 digit: all 8192 are candidates); at shift s, g of
    them have digit 1 and the rest 0; the bits below are random.
      g = 2048, K = 2048: the bin fills QW_SEL_MAX exactly: stop at s, ranked;
      g = 2049, K = 2049: cap 4096: stop at s, 2049 survivors sorted whole;
      g = 2049, K = 2048: the bin misses QW_SEL_MAX by one: the cut goes on to s - 8 (at s = 0: ties on the whole first
      word, sorted whole).
    Shift 56 only stops a cut whose candidates all survive: the level-0 radix digit spans the first 11 key bits, so every
    candidate's first byte reaches the K-th candidate's. There, 2048 candidates with K = 2047 are ranked and 4096 with
    K = 2049 sorted whole."""
    out = []
    for s in CUT_SHIFTS:
        order = DESC if (s // 8) % 2 == 0 else ASC
        variants = [(2048, 2048, "rank", s), (2049, 2049, "sort", s), (2049, 2048, "sort" if s == 0 else None, s)]
        if s == 56:
            variants = [(2048, 2047, "rank", 56), (4096, 2049, "sort", 56)]
        for g, K, branch, stop in variants:
            rng = random.Random(3000 + s * 7 + g + K)
            fillers = (0, 1, 2)
            nm = 8192 if s < 56 else g
            n = nm + 3
            matched = list(range(3, n))
            # s = 56: every candidate shares the level-0 digit (bits 63..53) and survives
            hi = (rng.getrandbits(63) | 1 << 63) >> min(s + 8, 53) << min(s + 8, 53)
            top = set(rng.sample(matched, g)) if s < 56 else set()
            va = {}
            for d in matched:
                if s < 56:
                    w = hi | (int(d in top) << s) | (rng.getrandbits(s) if s else 0)
                else:
                    w = hi | rng.getrandbits(53)
                r = (w & ~(1 << 63)) << 1 | rng.getrandbits(1)
                va[d] = _value(r, order)
            vals = {"a": (_filled(n, fillers, va), [True] * n)}
            tgt = {"n": nm}
            if branch is None:  # the bin misses QW_SEL_MAX by one: the cut resolves further digits
                tgt["stop_below"] = s
            else:
                tgt.update(stop=stop, branch=branch, m=g)
            out.append(Case(f"cut{s}-g{g}-K{K}", n, matched, vals, [("col", order, "a")], K, tgt))
    return out


EDGE_KS = [1, 2, 3, 4, 5, 1023, 1024, 1025, 2047, 2048, 2049, 3000, 4095, 4096]


def edge_cases() -> List[Case]:
    """K at every edge against matched counts K - 1, K, K + 1, 2048, 2049 and 8192 (random 64-bit values of a)."""
    out = []
    for K in EDGE_KS:
        for nm in sorted({K - 1, K, K + 1, 2048, 2049, 8192}):
            if nm < 1:
                continue
            rng = random.Random(4000 + K * 31 + nm)
            order = DESC if (K + nm) % 2 else ASC
            fillers = (0, 1, 2)
            n = nm + 3
            matched = list(range(3, n))
            va = {d: _value(rng.getrandbits(64), order) for d in matched}
            vals = {"a": (_filled(n, fillers, va), [True] * n)}
            tgt = {"m": nm} if nm <= K else {}
            out.append(Case(f"edge-K{K}-n{nm}", n, matched, vals, [("col", order, "a")], K, tgt))
    return out


def decode_cases() -> List[Case]:
    """write_hit layouts: an optional first column whose missing docs fall inside the top K (single key and first of
    two, both directions), the 1-doc split (doc_bits 0, a 0-bit column), doc-id sorts with doc_bits 11 and 12."""
    out = []
    for two in (False, True):
        for order in (DESC, ASC):
            rng = random.Random(5000 + 2 * two + order)
            fillers = (0, 1, 2)
            n = 1503
            matched = list(range(3, n))
            present = set(rng.sample(matched, 1000))
            va = {d: _value(rng.getrandbits(64), order) for d in present}
            ha = [d in present or d in fillers for d in range(n)]
            vb = {d: _value(rng.getrandbits(64), DESC) for d in matched}
            vals = {"a": (_filled(n, fillers, va), ha), "b": (_filled(n, fillers, vb), [True] * n)}
            sort = [("col", order, "a")] + ([("col", DESC, "b")] if two else [])
            out.append(Case(f"missing-{'ab' if two else 'a'}-{'d' if order == DESC else 'a'}", n, matched, vals, sort, 1200,
                            {"branch": "rank", "m": 1500, "common": 0}))
    for order in (DESC, ASC):
        for K in (1, 5):
            vals = {"a": ([12345], [True])}
            out.append(Case(f"one-doc-{'d' if order == DESC else 'a'}-K{K}", 1, [0], vals, [("col", order, "a")], K,
                            {"m": 1, "common": 192}))
            out.append(Case(f"one-doc-id-{'d' if order == DESC else 'a'}-K{K}", 1, [0], {}, [("doc", order, None)], K, {"m": 1}))
    for n in (2000, 4000):
        for order in (DESC, ASC):
            for K in (1000, 2048, 4096):
                matched = [d for d in range(n) if d % 97 != 5]
                out.append(Case(f"doc-n{n}-{'d' if order == DESC else 'a'}-K{K}", n, matched, {}, [("doc", order, None)], K))
    return [c for c in out]


def padding_cases() -> List[Case]:
    """sort_all_block with n far from a power of two: a DESC, b DESC, both optional; only 100 docs hold a value of a, so
    the rest tie on the first key word (w0 = 0) and every candidate survives. Doc 0 holds neither: its key is all zero,
    the value the sort pads with. K = 4096: for n = 2049 and 3000 the zero key is the last hit."""
    out = []
    for nm in (2049, 3000, 4097, 8191):
        rng = random.Random(6000 + nm)
        n = nm + 3
        fillers = (n - 3, n - 2, n - 1)
        matched = list(range(nm))
        with_a = set(rng.sample(range(1, nm), 100))
        with_b = set(rng.sample(range(1, nm), nm // 2))
        va = {d: rng.getrandbits(64) for d in with_a}
        vb = {d: rng.getrandbits(64) for d in with_b}
        ha = [d in with_a or d in fillers for d in range(n)]
        hb = [d in with_b or d in fillers for d in range(n)]
        vals = {"a": (_filled(n, fillers, va), ha), "b": (_filled(n, fillers, vb), hb)}
        out.append(Case(f"pad-n{nm}", n, matched, vals, [("col", DESC, "a"), ("col", DESC, "b")], 4096,
                        {"branch": "sort", "n": nm, "m": nm, "zero_key": True}))
    return out


def all_cases() -> Dict[str, List[Case]]:
    return {"at": at_cases((DESC, ASC)) + at_cases((ASC, DESC)), "cut": cut_cases(), "edge": edge_cases(),
            "decode": decode_cases(), "pad": padding_cases()}


# ---- _score on k_union -----------------------------------------------------------------------------------------------
class ScoreSplit:
    """n docs: term u in every doc, v in the top two score groups, all at tf 1 on a body field whose lengths set the
    group: g0 docs of length 1 with v score best, then g1 docs of length 2 with v; the rest (no v) have lengths 3..300.
    Column b: 64 bits (values 0, 1, 2^64 - 1 present); the two groups hold b < 2^40, so a `_score, b` key ties on its
    whole first word inside a group."""

    def __init__(self, n, g0, g1, seed):
        rng = np.random.default_rng(seed)
        d = np.arange(n)
        perm = rng.permutation(n)
        grp = np.full(n, 2)
        grp[perm[:g0]] = 0
        grp[perm[g0:g0 + g1]] = 1
        self.n, self.grp = n, grp
        self.lens = np.where(grp == 0, 1, np.where(grp == 1, 2, 3 + (d * 7919) % 298)).astype(np.int64)
        self.tf = {"u": np.ones(n, dtype=np.int64), "v": (grp < 2).astype(np.int64)}
        b = rng.integers(0, 1 << 40, size=n, dtype=np.uint64)
        rest = np.flatnonzero(grp == 2)
        b[rest[:3]] = np.array([0, 1, U64], dtype=np.uint64)
        self.b = Col(ffi.COL_U64, ffi.CARD_FULL, b, n)
        self.norm = bm25_norm(self.lens)

    def image(self, split_id):
        L = ffi.img_lib()
        uniq, inv = np.unique(self.lens, return_inverse=True)
        fn = np.array([L.qwgpu_fieldnorm_to_id(int(x)) for x in uniq], dtype=np.uint8)[inv]
        bld = S._Builder(self.n)
        body = bld.add_field("body", ffi.FIELD_HAS_FREQS | ffi.FIELD_HAS_FIELDNORMS, ffi.TOK_DEFAULT, fn, int(self.lens.sum()))
        for name in ("u", "v"):
            docs = np.flatnonzero(self.tf[name]).astype(np.uint32)
            bld.add_term(body, name.encode(), docs, self.tf[name][docs].astype(np.uint32))
        bld.add_column("b", ffi.COL_U64, ffi.CARD_FULL, self.b.vals, None)
        return bld.finish(split_id)

    def weights(self):
        return [np.float32(P.bm25_weight(int(np.count_nonzero(self.tf[t])), self.n)) for t in ("u", "v")]

    def scores(self) -> np.ndarray:
        s = np.zeros(self.n, dtype=np.float32)
        for t, w in zip(("u", "v"), self.weights()):
            s = (s + bm25_contributions(self.tf[t], self.norm, w)).astype(np.float32)
        return s

    def layout(self, with_b: bool, b_order: int = ASC) -> Layout:
        f = [("score", DESC, None)] + ([("col", b_order, self.b)] if with_b else [])
        return Layout(self.n, f, scores=self.scores(), scale=score_scale(self.weights()))

    def plan(self, img, K, with_b: bool, b_order: int = ASC) -> bytes:
        root = P.bool_([P.term(img, "body", t, occur=ffi.OCCUR_SHOULD) for t in ("u", "v")])
        sort = [(ffi.SORT_SCORE, DESC, ffi.ABSENT)] + ([(ffi.SORT_COLUMN, b_order, img.column_ord("b"))] if with_b else [])
        return P.make_plan(root, K, sort)


SCORE_KS = (2047, 2048, 2049)
SCORE_SPLITS = {"g2048": (20_000, 2048, 3000), "g2049": (20_000, 2049, 3000)}


def score_cases():
    """(name, ScoreSplit, K, with_b) for both splits, K in SCORE_KS, `_score` alone (QwScoreHit) and `_score, b ASC`."""
    out = []
    for sname, (n, g0, g1) in SCORE_SPLITS.items():
        sp = ScoreSplit(n, g0, g1, seed=g0)
        for K in SCORE_KS:
            for with_b in (False, True):
                out.append((f"score-{sname}-K{K}-{'sb' if with_b else 's'}", sp, K, with_b))
    return out
