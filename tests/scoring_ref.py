"""Expected results of term, union and phrase queries over a posting_corpora.Corpus, computed from the arrays the
split was built from.

Two restatements:
  * f32, bit-exact: helpers.bm25_contributions over the per-field norms (helpers.bm25_norm's arithmetic, from the
    fieldnorm ids and total_tokens), weights from the library's f32 idf (checked against numpy's within 1e-6), the
    clauses summed in plan order in f32. Expected: the match set, num_hits and the top K with identical f32 bits.
  * f64, independent: idf, k1 = 1.2, b = 0.75, the quantised fieldnorm and the average, all in f64, with its own
    error bound (`f64_bound`)."""
from __future__ import annotations

import ctypes as C
import math

import numpy as np

from quickwit_b200 import ffi, plan as P
from helpers import bm25_contributions, bm25_weight

K1, B = 1.2, 0.75
U = 2.0 ** -24


def _quant(ids):
    L = ffi.img_lib()
    table = np.array([L.qwgpu_id_to_fieldnorm(i) for i in range(256)], dtype=np.int64)
    return table[ids]


def norms(c, field):
    """Per-doc f32 BM25 length norm of `field`: helpers.bm25_norm's arithmetic from ids and total_tokens. A field
    without fieldnorms reads id 1 for every document."""
    key = ("_norm", field)
    if key not in c.__dict__:
        f = c.fields[field]
        ids = f.ids if f.ids is not None else np.ones(c.n, dtype=np.uint8)
        f32 = np.float32
        quant = _quant(ids).astype(np.float32)
        avg = f32(f.total_tokens) / f32(c.n)
        c.__dict__[key] = f32(K1) * (f32(1) - f32(B) + f32(B) * quant / avg)
    return c.__dict__[key]


def weight(c, field, term, boost=1.0):
    """The plan's f32 weight, checked against numpy's idf * (1 + k1) * boost."""
    df = len(c.postings[(field, term)][0])
    w = np.float32(P.bm25_weight(df, c.n, boost))
    ref = bm25_weight(df, c.n) * np.float32(boost)
    assert abs(float(w) - float(ref)) <= 1e-6 * abs(float(w)), (term, float(w), float(ref))
    return w


def phrase_counts(c, field, terms):
    """(docs, phrase counts) of a slop-0 phrase, from a scan of the position arrays."""
    per = []
    for t in terms:
        docs, tfs, pos = c.postings[(field, t)]
        starts = np.concatenate([[0], np.cumsum(tfs.astype(np.int64))])
        per.append({int(d): set(pos[starts[i]:starts[i + 1]].tolist()) for i, d in enumerate(docs)})
    common = sorted(set(per[0]).intersection(*per[1:]))
    out_d, out_c = [], []
    for d in common:
        cnt = sum(all(b + k in per[k][d] for k in range(1, len(terms))) for b in per[0][d])
        if cnt:
            out_d.append(d)
            out_c.append(cnt)
    return np.array(out_d, dtype=np.int64), np.array(out_c, dtype=np.uint32)


class Clause:
    """One scored clause: a term or a phrase of one field, with its boost."""

    def __init__(self, field, terms, boost=1.0):
        self.field, self.terms, self.boost = field, list(terms), boost

    def postings(self, c):
        if len(self.terms) == 1:
            docs, tfs, _ = c.postings[(self.field, self.terms[0])]
            return docs.astype(np.int64), tfs
        return phrase_counts(c, self.field, self.terms)

    def weight(self, c):
        if len(self.terms) == 1:
            return weight(c, self.field, self.terms[0], self.boost)
        f32 = np.float32
        dfs = [len(c.postings[(self.field, t)][0]) for t in self.terms]
        w = f32(ffi.img_lib().qwgpu_bm25_phrase_weight((C.c_uint64 * len(dfs))(*dfs), len(dfs), c.n, self.boost))
        idf = f32(0)
        for df in dfs:  # Bm25Weight::for_terms: the idfs summed in phrase order
            idf = idf + np.log(f32(1) + (f32(c.n - df) + f32(0.5)) / (f32(df) + f32(0.5)), dtype=np.float32)
        ref = idf * (f32(1) + f32(K1)) * f32(self.boost)
        assert abs(float(w) - float(ref)) <= 1e-6 * len(dfs) * abs(float(w)), (self.terms, float(w), float(ref))
        return w

    def idf64(self, c):
        return sum(math.log(1 + (c.n - len(c.postings[(self.field, t)][0]) + 0.5) / (len(c.postings[(self.field, t)][0]) + 0.5))
                   for t in self.terms)


def scores(c, clauses):
    """(match mask, f32 scores) of a union of `clauses`, summed in clause order."""
    s = np.zeros(c.n, dtype=np.float32)
    m = np.zeros(c.n, dtype=bool)
    for cl in clauses:
        docs, tfs = cl.postings(c)
        s[docs] = (s[docs] + bm25_contributions(tfs, norms(c, cl.field)[docs], cl.weight(c))).astype(np.float32)
        m[docs] = True
    return m, s


SORTS = {"score_desc": [(ffi.SORT_SCORE, ffi.ORDER_DESC, ffi.ABSENT)], "score_asc": [(ffi.SORT_SCORE, ffi.ORDER_ASC, ffi.ABSENT)],
         "doc_desc": [(ffi.SORT_DOCID, ffi.ORDER_DESC, ffi.ABSENT)], "doc_asc": [(ffi.SORT_DOCID, ffi.ORDER_ASC, ffi.ABSENT)]}
FILTER_MAX = 8  # the range filter f in [0, 8] over column f = doc % 10


def plan(c, clauses, K, sort="score_desc", must=None, filt=False):
    """Plan of a bool over `clauses` (SHOULD, or MUST for the clause at index `must`; every clause MUST when
    must == "all"), plus a FILTER range on column f when `filt`."""
    img = c.img
    kids = []
    for i, cl in enumerate(clauses):
        occ = ffi.OCCUR_MUST if must == "all" or i == must else ffi.OCCUR_SHOULD
        if len(cl.terms) == 1:
            kids.append(P.term(img, cl.field, cl.terms[0], occur=occ, boost=cl.boost))
        else:
            kids.append(P.phrase(img, cl.field, cl.terms, occur=occ, boost=cl.boost))
    if filt:
        kids.append(P.range_(img, "f", 0, FILTER_MAX, occur=ffi.OCCUR_FILTER))
    return P.make_plan(P.bool_(kids), K, SORTS[sort])


def expected(c, clauses, K, sort="score_desc", must=None, filt=False):
    """(num_hits, top-K doc ids, their f32 scores or None), for `plan`'s query.
    sort: score_desc (ties: doc desc), score_asc (ties: doc asc), doc_desc, doc_asc."""
    m, s = scores(c, clauses)
    for i, cl in enumerate(clauses):
        if must == "all" or i == must:
            req = np.zeros(c.n, dtype=bool)
            req[cl.postings(c)[0]] = True
            m &= req
    if filt:
        m &= np.asarray(c.columns["f"]) <= FILTER_MAX
    docs = np.flatnonzero(m)
    sc = s[docs]
    if sort == "score_desc":
        order = np.lexsort((-docs, -sc))
    elif sort == "score_asc":
        order = np.lexsort((docs, sc))
    elif sort == "doc_desc":
        order = np.argsort(-docs, kind="stable")
    else:
        order = np.argsort(docs, kind="stable")
    top = docs[order[:K]]
    return len(docs), top, (s[top] if sort.startswith("score") else None)


def scores64(c, clauses, docs):
    """f64 scores of `docs` from the raw quantities: idf, k1, b, quantised fieldnorm, total_tokens / num_docs."""
    out = np.zeros(len(docs), dtype=np.float64)
    for cl in clauses:
        f = c.fields[cl.field]
        cd, tfs = cl.postings(c)
        pos = np.searchsorted(cd, docs)
        hit = (pos < len(cd)) & (cd[np.minimum(pos, len(cd) - 1)] == docs)
        tf = np.where(hit, tfs[np.minimum(pos, len(cd) - 1)].astype(np.float64), 0.0)
        ids = f.ids[docs] if f.ids is not None else np.ones(len(docs), dtype=np.uint8)
        quant = _quant(ids).astype(np.float64)
        norm = K1 * (1 - B + B * quant / (f.total_tokens / c.n))
        out += np.where(hit, cl.idf64(c) * (1 + K1) * cl.boost * tf / (tf + norm), 0.0)
    return out


def f64_bound(c, clauses):
    """Relative bound on |f32 score - f64 score| for a union of `clauses` (u = 2^-24, every f32 op rounds once):
      weight  the idf argument 1 + (N - n + 0.5) / (n + 0.5) takes <= 4 roundings (N - n is exact: < 2^24 + 2^8),
              which log turns into an absolute error of 4u, i.e. 4u / idf relative, plus <= 2u from logf; an f32
              sum of k idfs (phrases) adds k u; times (1 + k1) (f32(1.2) and the sum: 2u) and times the boost (u).
      factor  tf / (tf + norm): the norm is k1 * (1 - b + b * q / avg) with avg = f32(total) / f32(N): total and
              the division, q / avg, b * x, the sum and k1 (whose f32 differs from 1.2 by u): <= 7u, which reaches
              the factor damped by norm / (tf + norm) < 1; f32(tf) (tf > 2^24), tf + norm and the division: 3u.
      product weight * factor: u.
    So every contribution is within (17 + k + 4k / idf_min) u of its exact value, and the f32 sum of c positive
    contributions in any order adds at most (c - 1) u of the total: the bound is (c + 16 + k + 4k / idf_min) u."""
    k = max(len(cl.terms) for cl in clauses)
    idf_min = min(min(math.log(1 + (c.n - len(c.postings[(cl.field, t)][0]) + 0.5) / (len(c.postings[(cl.field, t)][0]) + 0.5))
                      for t in cl.terms) for cl in clauses)
    return (len(clauses) + 16 + k + 4 * k / idf_min) * U


def check_f64(c, clauses, docs, got_scores, ctx=""):
    """Every f32 score within f64_bound of the f64 recomputation."""
    if len(docs) == 0:
        return
    want = scores64(c, clauses, np.asarray(docs, dtype=np.int64))
    got = np.asarray(got_scores, dtype=np.float32).astype(np.float64)
    rel = np.abs(got - want) / want
    bound = f64_bound(c, clauses)
    assert (rel <= bound).all(), f"{ctx}: f32 score off the f64 recomputation by {rel.max():.3g} > {bound:.3g} (doc {docs[int(np.argmax(rel))]})"


def check(got, c, clauses, K, sort="score_desc", must=None, filt=False, ctx=""):
    """A result (service.SplitSearchResult or oracle.OracleResult) of `plan(c, clauses, K, sort, must, filt)`
    against the f32 restatement, bit for bit, and, where scored, against the f64 bound."""
    nh, top, sc = expected(c, clauses, K, sort, must, filt)
    assert got.num_hits == nh, f"{ctx}: num_hits {got.num_hits} != {nh}"
    gd = [h[0] for h in got.hits]
    if gd != top.tolist():
        i = next((i for i, (a, b) in enumerate(zip(gd, top.tolist())) if a != b), min(len(gd), len(top)))
        raise AssertionError(f"{ctx}: hit {i} differs: got {gd[i:i + 3]} want {top[i:i + 3].tolist()} (n={len(gd)}/{len(top)})")
    if sc is not None:
        gs = np.array([h[4] for h in got.hits], dtype=np.float32)
        assert np.array_equal(gs.view(np.uint32), sc.view(np.uint32)), f"{ctx}: f32 score bits differ from the restatement"
        check_f64(c, clauses, top, gs, ctx)


def phrase_prefix_docs(c, field, exact, prefix):
    """Docs where `exact` sits at some b and a term of `field` starting with `prefix` at b + 1, from the positions."""
    out = set()
    for (f, t) in c.postings:
        if f == field and t.startswith(prefix):
            out.update(phrase_counts(c, field, [exact, t])[0].tolist())
    return np.array(sorted(out), dtype=np.int64)
