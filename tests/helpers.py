"""Shared test helpers: plan/agg construction against a split image, result comparison."""
from __future__ import annotations

import math
from typing import List, Sequence

import numpy as np

from quickwit_b200 import ffi, plan as P, splitgen as S

SCORE_DESC = [(ffi.SORT_SCORE, ffi.ORDER_DESC, ffi.ABSENT)]
DOC_DESC = [(ffi.SORT_DOCID, ffi.ORDER_DESC, ffi.ABSENT)]
DOC_ASC = [(ffi.SORT_DOCID, ffi.ORDER_ASC, ffi.ABSENT)]


def col_sort(img, name, order):
    c = img.column_ord(name)
    return (ffi.SORT_COLUMN, order, c if c >= 0 else ffi.ABSENT)


def mapped_to_f64(ctype: int, m: int) -> float:
    if ctype in (ffi.COL_U64, ffi.COL_BOOL, ffi.COL_STR):
        return float(m)
    if ctype in (ffi.COL_I64, ffi.COL_DATETIME):
        return float(S.u64_to_i64(m))
    return S.u64_to_f64(m)


def histogram_agg(img, column: str, interval: float, offset: float = 0.0, children=(), bounds=None) -> P.Agg:
    c = img.column_ord(column)
    col = img.columns()[c]
    lo = mapped_to_f64(col.type, col.min_value)
    hi = mapped_to_f64(col.type, col.max_value)
    base = math.floor((lo - offset) / interval)
    top = math.floor((hi - offset) / interval)
    return P.Agg(ffi.AGG_HISTOGRAM, column=c, num_buckets=int(top - base + 1), interval=interval, offset=offset,
                 base_pos=int(base), children=children, bounds=bounds)


def terms_agg(img, column: str, children=(), missing=None) -> P.Agg:
    c = img.column_ord(column)
    if c < 0:
        return P.Agg(ffi.AGG_TERMS, column=ffi.ABSENT, num_buckets=1 if missing is not None else 0, children=children,
                     missing=missing)
    col = img.columns()[c]
    nb = (col.max_value - col.min_value) // col.gcd + 1
    return P.Agg(ffi.AGG_TERMS, column=c, num_buckets=int(nb) + (1 if missing is not None else 0), children=children,
                 missing=missing)


def stats_agg(img, column: str) -> P.Agg:
    c = img.column_ord(column)
    return P.Agg(ffi.AGG_STATS, column=c if c >= 0 else ffi.ABSENT)


def range_agg(img, column: str, ranges) -> P.Agg:
    c = img.column_ord(column)
    return P.Agg(ffi.AGG_RANGE, column=c, num_buckets=len(ranges), ranges=ranges)


def bm25_norm(lengths: np.ndarray) -> np.ndarray:
    """Per-doc BM25 length norm restated in numpy float32 (tantivy Bm25Weight; formula verified against the reference
    golden in SURVEY.md Appendix B.1): k1 * (1 - b + b * fieldnorm / avg_fieldnorm), with the fieldnorm QUANTISED through
    the 256-entry id table and avg_fieldnorm = total tokens / number of docs."""
    L = ffi.img_lib()
    lengths = np.asarray(lengths, dtype=np.int64)
    uniq, inv = np.unique(lengths, return_inverse=True)
    quant = np.array([L.qwgpu_id_to_fieldnorm(L.qwgpu_fieldnorm_to_id(int(x))) for x in uniq], dtype=np.float32)[inv]
    f32 = np.float32
    avg = f32(lengths.sum()) / f32(len(lengths))
    k1, b = f32(1.2), f32(0.75)
    return k1 * (f32(1) - b + b * quant / avg)


def bm25_weight(doc_freq: int, num_docs: int) -> np.float32:
    """idf * (1 + k1) in float32, idf = ln(1 + (N - n + 0.5) / (n + 0.5))."""
    f32 = np.float32
    idf = np.log(f32(1) + (f32(num_docs - doc_freq) + f32(0.5)) / (f32(doc_freq) + f32(0.5)), dtype=np.float32)
    return idf * (f32(1) + f32(1.2))


def bm25_contributions(tf: np.ndarray, norm: np.ndarray, weight) -> np.ndarray:
    """One term's per-doc score, weight * (tf / (tf + norm)), 0 where the term is absent (tf == 0). A union adds the
    contributions of its clauses in clause order, in float32."""
    tf = np.asarray(tf, dtype=np.float32)
    with np.errstate(invalid="ignore"):
        return np.where(tf > 0, np.float32(weight) * (tf / (tf + norm)), np.float32(0)).astype(np.float32)


def assert_same(got, want, f64_sum_cells: Sequence[int] = (), ctx: str = ""):
    """got: service.SplitSearchResult, want: oracle.OracleResult. Bit-exact everywhere (doc ids,
    sort values, f32 score bits, counts); f64 sums of f64 columns within 1e-9 relative."""
    assert got.num_hits == want.num_hits, f"{ctx}: num_hits {got.num_hits} != {want.num_hits}"
    g = [(h[0], h[1], h[2], h[3]) for h in got.hits]
    w = [(h[0], h[1], h[2], h[3]) for h in want.hits]
    if g != w:
        for i, (a, b) in enumerate(zip(g, w)):
            if a != b:
                raise AssertionError(f"{ctx}: hit {i} differs: gpu {a} oracle {b} (n={len(g)}/{len(w)})")
        raise AssertionError(f"{ctx}: hit count {len(g)} != {len(w)}")
    gs = np.array([h[4] for h in got.hits], dtype=np.float32).view(np.uint32)
    ws_ = np.array([h[4] for h in want.hits], dtype=np.float32).view(np.uint32)
    assert np.array_equal(gs, ws_), f"{ctx}: f32 score bits differ"
    assert len(got.cells) == len(want.cells), f"{ctx}: cell count {len(got.cells)} != {len(want.cells)}"
    for i, (a, b) in enumerate(zip(got.cells, want.cells)):
        if i in f64_sum_cells:
            assert a[0] == b[0] and a[2:] == b[2:], f"{ctx}: cell {i}: {a} != {b}"
            fa, fb = S.struct.unpack("<d", S.struct.pack("<Q", a[1]))[0], S.struct.unpack("<d", S.struct.pack("<Q", b[1]))[0]
            assert abs(fa - fb) <= 1e-9 * max(1.0, abs(fb)), f"{ctx}: cell {i} f64 sum {fa} vs {fb}"
        else:
            assert a == b, f"{ctx}: cell {i}: gpu {a} != oracle {b}"
