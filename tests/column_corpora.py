"""Splits for the fast-field filter and sort-key tests, built column by column from numpy arrays that column_ref reads
back (never the image): a FULL u64 column per bit-packed width 0..64, OPTIONAL and MULTI copies at the widths where
the packed reads change shape, gcd columns, the type edges of every mapped type, and a raw text field whose terms
drive the plan onto k_driver and k_window's candidate gather."""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from quickwit_b200 import ffi, splitgen as S

U64_MAX = (1 << 64) - 1
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


class Col:
    """A column as the split was built from it: mapped-u64 values in index order and the doc of each value.
    card FULL: value d belongs to doc d; OPTIONAL: one value per present doc; MULTI: `start` (num_docs + 1 offsets)."""

    def __init__(self, ctype: int, card: int, vals, num_docs: int, docs=None, start=None):
        self.ctype, self.card, self.num_docs = ctype, card, num_docs
        self.vals = np.ascontiguousarray(vals, dtype=np.uint64)
        if card == ffi.CARD_FULL:
            assert self.vals.size == num_docs
            self.doc_of = np.arange(num_docs, dtype=np.int64)
        elif card == ffi.CARD_OPTIONAL:
            self.doc_of = np.asarray(docs, dtype=np.int64)
            assert self.doc_of.size == self.vals.size and np.all(np.diff(self.doc_of) > 0)
        else:
            self.start = np.asarray(start, dtype=np.int64)
            assert self.start.size == num_docs + 1 and self.start[-1] == self.vals.size
            self.doc_of = np.repeat(np.arange(num_docs, dtype=np.int64), np.diff(self.start))
        self.num_vals = int(self.vals.size)
        self.min = int(self.vals.min()) if self.num_vals else 0
        self.max = int(self.vals.max()) if self.num_vals else 0
        self.gcd = (int(np.gcd.reduce(self.vals - np.uint64(self.min))) if self.num_vals else 0) or 1
        self.bits = ((self.max - self.min) // self.gcd).bit_length()
        # the doc's first value in index order (its sort value), and whether it has one
        self.has = np.zeros(num_docs, dtype=bool)
        self.has[self.doc_of] = True
        self.first = np.zeros(num_docs, dtype=np.uint64)
        first_idx = np.unique(self.doc_of, return_index=True)[1]
        self.first[self.doc_of[first_idx]] = self.vals[first_idx]

    def index(self) -> Optional[np.ndarray]:
        if self.card == ffi.CARD_FULL:
            return None
        return (self.doc_of if self.card == ffi.CARD_OPTIONAL else self.start).astype(np.uint32)


class Split:
    """One split image: the columns, and the raw-tokenized text field `t` whose terms are `terms[name]` (sorted doc
    ids)."""

    def __init__(self, split_id: str, num_docs: int, cols: Sequence[Tuple[str, Col]], terms: Dict[str, np.ndarray]):
        b = S._Builder(num_docs)
        fid = b.add_field("t", 0, ffi.TOK_RAW, None, int(sum(len(d) for d in terms.values())))
        for name in sorted(terms):
            b.add_term(fid, name.encode(), terms[name], None)
        for name, c in cols:
            assert c.num_docs == num_docs, name
            b.add_column(name, c.ctype, c.card, c.vals, c.index())
        self.img = b.finish(split_id)
        self.split_id, self.num_docs = split_id, num_docs
        self.cols: Dict[str, Col] = dict(cols)
        self.terms = {k: np.asarray(v, dtype=np.int64) for k, v in terms.items()}
        self.ords = {name: self.img.column_ord(name) for name, _ in cols}


def span_raws(n: int, b: int, rng: np.random.Generator) -> np.ndarray:
    """n raws spanning exactly b bits: 0, 1 and 2^b - 1 present (the gcd stays 1), a third of them drawn from a pool of
    16 values (ties the sort must break by doc id), the rest uniform."""
    if b == 0:
        return np.zeros(n, dtype=np.uint64)
    top = (1 << b) - 1
    r = rng.integers(0, 1 << 63, size=n, dtype=np.uint64, endpoint=True) if b == 64 else \
        rng.integers(0, top, size=n, dtype=np.uint64, endpoint=True)
    if b == 64:
        r = (r << np.uint64(1)) | rng.integers(0, 2, size=n, dtype=np.uint64)
    pool = r[rng.integers(0, n, size=16)]
    tie = rng.random(n) < 1 / 3
    r[tie] = pool[rng.integers(0, 16, size=int(tie.sum()))]
    fixed = [0, 1, top, 1 if b > 1 else 0, top]
    for i, v in zip((n // 7, n // 3, n - 1, 0, n // 2), fixed):
        r[i % n] = v
    if n >= 3:
        r[1], r[2] = 0, top
    return r


def _base(b: int) -> int:
    return 0 if b == 64 else 5


# ---- the main split ---------------------------------------------------------------------------------------------
N_MAIN = 40_037                    # not a multiple of 32, 64 or the 32768-doc k_window window; two windows
MC_WIDTHS = (0, 1, 9, 10, 11, 31, 32, 33, 53, 63, 64)
G1000_MIN, G3_MIN = 10**15 + 17, (1 << 40) + 1
F64_EDGES = [-math.inf, -1.7976931348623157e308, -1e-300, -0.0, 0.0, 5e-324, 1.7976931348623157e308, math.inf,
             math.nan]
I64_EDGES = [I64_MIN, -1, 0, I64_MAX]
U64_EDGES = [1 << 63, (1 << 63) + 1, U64_MAX - 1, U64_MAX, 0, 3]
STEP = 1024                        # the candidate gather's step: 32 bitmap words


def _optional_present(n: int, rng: np.random.Generator, flip: bool) -> np.ndarray:
    """~60 % present; docs 63 and 127 present and 64 and 128 absent (or the other way round with `flip`), the last doc
    present unless `flip`."""
    p = rng.random(n) < 0.6
    for d in (63, 127):
        p[d] = not flip
    for d in (64, 128):
        p[d] = flip
    p[n - 1] = not flip
    p[0] = flip
    return p


def _multi_counts(n: int, rng: np.random.Generator) -> np.ndarray:
    """0..4 values per doc; docs 63 / 64 / 127 / the last doc with 0, 1, 4 and 0 values."""
    c = rng.integers(0, 5, size=n)
    c[63], c[64], c[127], c[n - 1] = 0, 1, 4, 0
    return c


def _driving_terms(n: int, rng: np.random.Generator) -> Dict[str, np.ndarray]:
    """`all`; `d30` (~30 %); `sparse` (3 docs in each 1024-doc step); `q128` / `q129`: exactly 128 docs in step 1 and
    129 docs in step 2 (the gather's sparse and dense paths), and 5 docs in every other step."""
    docs = np.arange(n)
    t = {"all": docs, "d30": docs[rng.random(n) < 0.3]}
    steps = range(0, n, STEP)
    t["sparse"] = np.unique(np.concatenate([s + rng.choice(min(STEP, n - s), 3, replace=False) for s in steps]))
    for name, (k_step, k) in (("q128", (1, 128)), ("q129", (2, 129))):
        parts = []
        for si, s in enumerate(steps):
            m = min(STEP, n - s)
            parts.append(s + rng.choice(m, k if si == k_step else min(5, m), replace=False))
        t[name] = np.unique(np.concatenate(parts))
    return {k: np.sort(v).astype(np.int64) for k, v in t.items()}


def main_split(split_id: str = "cf-main", seed: int = 17) -> Split:
    n = N_MAIN
    rng = np.random.default_rng(seed)
    cols: List[Tuple[str, Col]] = []
    for b in range(65):
        cols.append((f"w{b}", Col(ffi.COL_U64, ffi.CARD_FULL, _base(b) + span_raws(n, b, rng), n)))
    for i, b in enumerate(MC_WIDTHS):
        p = _optional_present(n, rng, flip=bool(i % 2))
        docs = np.nonzero(p)[0]
        cols.append((f"o{b}", Col(ffi.COL_U64, ffi.CARD_OPTIONAL, _base(b) + span_raws(docs.size, b, rng), n, docs=docs)))
        cnt = _multi_counts(n, rng)
        start = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(cnt, out=start[1:])
        cols.append((f"m{b}", Col(ffi.COL_U64, ffi.CARD_MULTI, _base(b) + span_raws(int(start[-1]), b, rng), n, start=start)))
    # gcd 1000 with a min far from 0, gcd 3
    cols.append(("g1000", Col(ffi.COL_U64, ffi.CARD_FULL, G1000_MIN + 1000 * rng.integers(0, 5000, size=n).astype(np.uint64), n)))
    cols.append(("g3", Col(ffi.COL_U64, ffi.CARD_FULL, G3_MIN + 3 * rng.integers(0, 1 << 20, size=n).astype(np.uint64), n)))
    # type edges, in mapped space
    iv = rng.integers(I64_MIN, I64_MAX, size=n, dtype=np.int64, endpoint=True)
    iv[rng.random(n) < 0.3] = rng.integers(-5, 6, size=1)[0]
    for k, v in enumerate(I64_EDGES):
        iv[17 * k + 3::N_MAIN // 7] = v
    cols.append(("i64", Col(ffi.COL_I64, ffi.CARD_FULL, [S.i64_to_u64(int(x)) for x in iv], n)))
    uv = rng.integers(1 << 63, U64_MAX, size=n, dtype=np.uint64, endpoint=True)
    for k, v in enumerate(U64_EDGES):
        uv[11 * k + 5::N_MAIN // 5] = v
    cols.append(("u64", Col(ffi.COL_U64, ffi.CARD_FULL, uv, n)))
    p = _optional_present(n, rng, flip=False)
    fdocs = np.nonzero(p)[0]
    fv = rng.normal(0.0, 1e3, size=fdocs.size)
    fv[rng.random(fdocs.size) < 0.2] = 0.5
    for k, v in enumerate(F64_EDGES):
        fv[13 * k + 1::fdocs.size // 9] = v
    cols.append(("f64", Col(ffi.COL_F64, ffi.CARD_OPTIONAL, [S.f64_to_u64(float(x)) for x in fv], n, docs=fdocs)))
    ns = rng.integers(-2 * 10**18, 10**18, size=n, dtype=np.int64)
    ns[rng.random(n) < 0.25] = -1
    cols.append(("dt", Col(ffi.COL_DATETIME, ffi.CARD_FULL, [S.i64_to_u64(int(x)) for x in ns], n)))
    bo = (rng.random(n) < 0.4).astype(np.uint64)
    cols.append(("bool", Col(ffi.COL_BOOL, ffi.CARD_FULL, bo, n)))
    return Split(split_id, n, cols, _driving_terms(n, rng))


# ---- small splits: 1 doc (doc_bits 0), 1024, 2048 and 2049 docs (doc_bits 10, 11, 12: the edge of QW_TOP_DOC) ------
SMALL_DOCS = (1, 1024, 2048, 2049)
SMALL_WIDTHS = (0, 3, 10, 33, 64)


def small_split(n: int, seed: int = 5) -> Split:
    rng = np.random.default_rng(seed + n)
    cols: List[Tuple[str, Col]] = []
    for b in SMALL_WIDTHS:
        raws = span_raws(n, b, rng) if n > 2 else np.full(n, (1 << b) - 1 if b < 64 else U64_MAX, dtype=np.uint64)
        cols.append((f"w{b}", Col(ffi.COL_U64, ffi.CARD_FULL, (_base(b) + raws) if n > 2 else raws, n)))
    p = rng.random(n) < 0.5
    p[-1] = True
    docs = np.nonzero(p)[0]
    cols.append(("o10", Col(ffi.COL_U64, ffi.CARD_OPTIONAL, 5 + span_raws(docs.size, 10, rng) if docs.size > 2 else
                            np.full(docs.size, 1000, dtype=np.uint64), n, docs=docs)))
    terms = {"all": np.arange(n), "d30": np.nonzero(rng.random(n) < 0.3)[0]}
    if terms["d30"].size == 0:
        terms["d30"] = np.array([n - 1])
    return Split(f"cf-small-{n}", n, cols, terms)


# ---- the splits of the device-merge test: the same fields with a different width, min and gcd in each --------------
MERGE_MAPPING = {"field_mappings": [{"name": "body", "type": "text", "tokenizer": "raw"},
                                    {"name": "u", "type": "u64", "fast": True},
                                    {"name": "i", "type": "i64", "fast": True},
                                    {"name": "f", "type": "f64", "fast": True}]}


def merge_docs(seed: int = 23) -> List[List[dict]]:
    """Five splits' documents. u: 0..5 / >= 2^63 / multiples of 1000 / wide / absent from a whole split; i and f
    likewise change their range from split to split; about 15 % of docs miss each field."""
    rng = np.random.default_rng(seed)
    sizes = (300, 257, 411, 129, 200)
    u_gen = [lambda: int(rng.integers(0, 6)),
             lambda: int(rng.integers(1 << 63, U64_MAX, dtype=np.uint64, endpoint=True)),
             lambda: 1000 * int(rng.integers(0, 40)) + 7_000_000,
             lambda: int(rng.integers(0, 1 << 62)) if rng.random() < 0.5 else int(rng.integers(0, 6)),
             None]
    i_gen = [lambda: int(rng.integers(-3, 4)), lambda: int(rng.integers(I64_MIN, I64_MAX, endpoint=True)),
             lambda: -1000 * int(rng.integers(0, 50)), lambda: int(rng.integers(0, 3)), lambda: int(rng.integers(-3, 4))]
    f_gen = [lambda: float(rng.integers(-4, 5)) / 2, lambda: float(rng.normal(0, 1e12)),
             lambda: float(rng.choice([-0.0, 0.0, 1.5, -1.5, math.inf, -math.inf])), lambda: 0.25,
             lambda: float(rng.uniform(-1, 1))]
    out = []
    for s, n in enumerate(sizes):
        docs = []
        for _ in range(n):
            d = {"body": "x" if rng.random() < 0.7 else "y"}
            if u_gen[s] is not None and rng.random() < 0.85:
                d["u"] = u_gen[s]()
            if rng.random() < 0.85:
                d["i"] = i_gen[s]()
            if rng.random() < 0.85:
                d["f"] = f_gen[s]()
            docs.append(d)
        out.append(docs)
    return out


def merge_splits(docs: Sequence[Sequence[dict]]) -> list:
    return [S.build_split(list(d), MERGE_MAPPING, f"cf-merge-{i}") for i, d in enumerate(docs)]
