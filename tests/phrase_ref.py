"""The phrase, phrase-prefix and term-set results of a phrase_corpora corpus, restated from the arrays the split was
built from (docs, tfs and positions per term; fieldnorm ids and total_tokens per field), never from the image.

  * Phrase count (tantivy's rule, any offsets): the number of integers c, in Python's unbounded ints, such that every
    term k has a position at c + lo_k. c may be negative: offsets (1, 2) over "a b" match at c = -1.
  * Phrase prefix: the docs where some c has every exact term i at c + lo_i and some expansion at c + lo_last.
  * Term set: the union of the terms' doc lists.
  * Phrase score: f32 weight * (count / (count + norm)), the weight Bm25Weight::for_terms through the library (checked
    against numpy by scoring_ref.Clause.weight), the norm scoring_ref.norms' arithmetic.
A bool over such clauses adds its scored MUST contributions in plan order, then its SHOULD contributions, as the
window program does (msum + ssum)."""
from __future__ import annotations

import numpy as np

from quickwit_b200 import ffi, plan as P
from helpers import bm25_contributions
import scoring_ref as R

MUST, SHOULD, FILTER, MUST_NOT = ffi.OCCUR_MUST, ffi.OCCUR_SHOULD, ffi.OCCUR_FILTER, ffi.OCCUR_MUST_NOT


def term_ord(img, field, term):
    """img.term_ord through a dictionary built once per image and field (img.term_ord scans the field's terms)."""
    cache = img.__dict__.setdefault("_ords", {})
    if field not in cache:
        _h, _s, tbytes, fields, terms, _c = img._directory()
        f = fields[img.field_names().index(field)]
        cache[field] = {bytes(tbytes[terms[t].bytes_off: terms[t].bytes_off + terms[t].bytes_len]).decode(): t
                        for t in range(f.first_term, f.first_term + f.num_terms)}
    return cache[field].get(term, -1)


def _keys(c, field, term, lo, docs):
    """int64 keys doc * 2^34 + (position - lo + 2^33) of `term`'s positions in `docs` (sorted, unique)."""
    d, tfs, pos = c.postings[(field, term)]
    keep = np.isin(d, docs)
    owner = np.repeat(np.arange(len(d)), tfs.astype(np.int64))
    sel = keep[owner]
    return np.sort(d.astype(np.int64)[owner[sel]] * (1 << 34) + (pos[sel].astype(np.int64) - int(lo) + (1 << 33)))


def _memo(c, key, fn):
    memo = c.__dict__.setdefault("_phrase_ref", {})
    if key not in memo:
        memo[key] = fn()
    return memo[key]


def _aligned(c, field, groups, offsets):
    """Keys c of the alignment constants at which every group (a list of terms: any of them) has a position at
    c + offsets[k], within the docs every group holds."""
    docs = None
    for g in groups:
        gd = np.unique(np.concatenate([c.postings[(field, t)][0] for t in g]))
        docs = gd if docs is None else np.intersect1d(docs, gd)
    keys = None
    for g, lo in zip(groups, offsets):
        k = np.unique(np.concatenate([_keys(c, field, t, lo, docs) for t in g]))
        keys = k if keys is None else np.intersect1d(keys, k, assume_unique=True)
    return keys


def phrase_counts(c, field, terms, offsets):
    """(docs int64, counts uint32) of a slop-0 phrase whose term k sits at offset offsets[k]."""
    def run():
        d, n = np.unique(_aligned(c, field, [[t] for t in terms], offsets) >> 34, return_counts=True)
        return d.astype(np.int64), n.astype(np.uint32)
    return _memo(c, ("phrase", field, tuple(terms), tuple(offsets)), run)


def prefix_docs(c, field, exact, offsets, expansions, exp_offset):
    """Docs of a phrase prefix: exact terms at `offsets`, any of `expansions` at `exp_offset`."""
    def run():
        keys = _aligned(c, field, [[t] for t in exact] + [list(expansions)], list(offsets) + [exp_offset])
        return np.unique(keys >> 34).astype(np.int64)
    return _memo(c, ("prefix", field, tuple(exact), tuple(offsets), tuple(expansions), exp_offset), run)


def term_set_docs(c, field, terms):
    return _memo(c, ("set", field, tuple(terms)),
                 lambda: np.unique(np.concatenate([c.postings[(field, t)][0] for t in terms])).astype(np.int64))


class Phrase:
    """A PHRASE node with explicit offsets (default 0..k-1)."""
    kind = "phrase"

    def __init__(self, field, terms, offsets=None, occur=MUST, boost=1.0):
        self.field, self.terms = field, list(terms)
        self.offsets = list(range(len(terms))) if offsets is None else list(offsets)
        self.occur, self.boost = occur, boost

    def node(self, img):
        fid = img.field_names().index(self.field)
        ords = [term_ord(img, self.field, t) for t in self.terms]
        assert all(o >= 0 for o in ords), self.terms
        kids = [P.Node(ffi.NODE_TERM, MUST, 1.0, term_ord=o, field_id=fid, weight=P.bm25_weight(img.doc_freq(o), img.num_docs), lo=lo)
                for o, lo in zip(ords, self.offsets)]
        return P.Node(ffi.NODE_PHRASE, self.occur, self.boost, children=kids, field_id=fid, weight=float(self.weight(None, img)))

    def weight(self, c, img=None):
        if c is not None:
            return R.Clause(self.field, self.terms, self.boost).weight(c)
        import ctypes as C
        dfs = [img.doc_freq(term_ord(img, self.field, t)) for t in self.terms]
        return np.float32(ffi.img_lib().qwgpu_bm25_phrase_weight((C.c_uint64 * len(dfs))(*dfs), len(dfs), img.num_docs, self.boost))

    def matches(self, c):
        return phrase_counts(c, self.field, self.terms, self.offsets)

    def contributions(self, c, docs, counts):
        return bm25_contributions(counts, R.norms(c, self.field)[docs], self.weight(c))

    def label(self):
        return f"{self.field}:{'/'.join(self.terms[:3])}{'..' if len(self.terms) > 3 else ''}({len(self.terms)})@{self.offsets[:4]}"


class Prefix:
    """A PHRASE_PREFIX node: `exact` at `offsets`, then `expansions` (term names) at `exp_offset`. Never scored."""
    kind = "prefix"

    def __init__(self, field, exact, expansions, offsets=None, exp_offset=None, occur=MUST):
        self.field, self.exact, self.expansions = field, list(exact), list(expansions)
        self.offsets = list(range(len(exact))) if offsets is None else list(offsets)
        self.exp_offset = len(exact) if exp_offset is None else exp_offset
        self.occur = occur

    def node(self, img):
        fid = img.field_names().index(self.field)

        def kid(t, lo):
            o = term_ord(img, self.field, t)
            assert o >= 0, t
            return P.Node(ffi.NODE_TERM, MUST, 1.0, term_ord=o, field_id=fid, weight=P.bm25_weight(img.doc_freq(o), img.num_docs), lo=lo)

        kids = [kid(t, lo) for t, lo in zip(self.exact, self.offsets)] + [kid(t, self.exp_offset) for t in self.expansions]
        return P.Node(ffi.NODE_PHRASE_PREFIX, self.occur, children=kids, field_id=fid, lo=len(self.exact))

    def matches(self, c):
        d = prefix_docs(c, self.field, self.exact, self.offsets, self.expansions, self.exp_offset)
        return d, np.ones(len(d), dtype=np.uint32)

    def label(self):
        return f"prefix {self.field}:{'/'.join(self.exact[:3])}({len(self.exact)}) + {len(self.expansions)} exp @{self.offsets[:4]},{self.exp_offset}"


class TermSet:
    """A TERM_SET node over term names of one field. Never scored."""
    kind = "term_set"

    def __init__(self, field, terms, occur=FILTER):
        self.field, self.terms, self.occur = field, list(terms), occur

    def node(self, img):
        return P.term_set(img, self.field, sorted(term_ord(img, self.field, t) for t in self.terms), occur=self.occur)

    def matches(self, c):
        d = term_set_docs(c, self.field, self.terms)
        return d, np.ones(len(d), dtype=np.uint32)

    def label(self):
        return f"term set {self.field}:{self.terms[0]}..({len(self.terms)})"


class Term:
    """A plain TERM clause (beside a phrase in a bool)."""
    kind = "term"

    def __init__(self, field, term, occur=SHOULD):
        self.field, self.term, self.occur = field, term, occur

    def node(self, img):
        return P.term(img, self.field, self.term, occur=self.occur)

    def matches(self, c):
        d, tfs, _ = c.postings[(self.field, self.term)]
        return d.astype(np.int64), tfs

    def contributions(self, c, docs, tfs):
        return bm25_contributions(tfs, R.norms(c, self.field)[docs], R.weight(c, self.field, self.term))

    def label(self):
        return f"term {self.field}:{self.term}"


SORTS = {"score_desc": R.SORTS["score_desc"], "doc_asc": R.SORTS["doc_asc"], "doc_desc": R.SORTS["doc_desc"]}


def evaluate(c, clauses, msm, scoring):
    """(match mask, f32 scores) of a bool over `clauses` with minimum_should_match `msm`: scored MUST contributions
    summed in plan order, then the SHOULD ones, then the two sums added (the window program's msum + ssum). A nested
    bool contributes its own score."""
    n = c.n
    req = np.ones(n, dtype=bool)
    nsh = np.zeros(n, dtype=np.int64)
    ban = np.zeros(n, dtype=bool)
    msum = np.zeros(n, dtype=np.float32)
    ssum = np.zeros(n, dtype=np.float32)
    n_req = 0
    for cl in clauses:
        scored = scoring and cl.occur in (MUST, SHOULD)
        if cl.kind == "bool":
            m, sub = evaluate(c, cl.clauses, cl.msm, scored)
            docs = np.flatnonzero(m)
            contrib = sub[docs]
        else:
            docs, vals = cl.matches(c)
            m = np.zeros(n, dtype=bool)
            m[docs] = True
            contrib = cl.contributions(c, docs, vals) if scored and cl.kind in ("phrase", "term") else None
        if cl.occur in (MUST, FILTER):
            req &= m
            n_req += 1
        elif cl.occur == SHOULD:
            nsh += m
        else:
            ban |= m
        if contrib is not None and scored:
            acc = msum if cl.occur == MUST else ssum
            acc[docs] = (acc[docs] + contrib).astype(np.float32)
    need = msm if msm else (0 if n_req else 1)
    return req & (nsh >= need) & ~ban, (msum + ssum).astype(np.float32)


class Bool:
    """A nested BOOL clause."""
    kind = "bool"

    def __init__(self, clauses, occur=MUST, msm=None):
        self.clauses, self.occur, self.msm = list(clauses), occur, msm

    def node(self, img):
        return P.bool_([cl.node(img) for cl in self.clauses], min_should_match=self.msm, occur=self.occur)

    def label(self):
        return "(" + " & ".join(f"{cl.label()}[{cl.occur}]" for cl in self.clauses) + ")"


class Query:
    """One plan: a bool over `clauses` (each carries its occur) with `msm`, or the lone clause itself when `bare`."""

    def __init__(self, clauses, msm=None, bare=False):
        self.clauses, self.msm, self.bare = list(clauses), msm, bare and len(clauses) == 1

    def root(self, img):
        if self.bare:
            return self.clauses[0].node(img)
        return P.bool_([cl.node(img) for cl in self.clauses], min_should_match=self.msm)

    def plan(self, img, K, sort="score_desc"):
        return P.make_plan(self.root(img), K, SORTS[sort])

    def expected(self, c, K, sort="score_desc"):
        """(num_hits, top-K doc ids, their f32 scores or None)."""
        scoring = sort == "score_desc"
        match, s = evaluate(c, self.clauses, self.msm, scoring)
        docs = np.flatnonzero(match)
        if sort == "score_desc":
            order = np.lexsort((-docs, -s[docs]))
        elif sort == "doc_desc":
            order = np.argsort(-docs, kind="stable")
        else:
            order = np.argsort(docs, kind="stable")
        top = docs[order[:K]]
        return len(docs), top, (s[top] if scoring else None)

    def label(self):
        return " & ".join(f"{cl.label()}[{cl.occur}]" for cl in self.clauses) + (f" msm={self.msm}" if self.msm else "")


def check(got, c, q, K, sort, ctx=""):
    """A result (service.SplitSearchResult or oracle.OracleResult) of q.plan(img, K, sort) against the restatement:
    num_hits, doc ids and f32 score bits."""
    nh, top, sc = q.expected(c, K, sort)
    assert got.num_hits == nh, f"{ctx}: num_hits {got.num_hits} != {nh}"
    gd = [h[0] for h in got.hits]
    if gd != top.tolist():
        i = next((i for i, (a, b) in enumerate(zip(gd, top.tolist())) if a != b), min(len(gd), len(top)))
        raise AssertionError(f"{ctx}: hit {i} differs: got {gd[i:i + 3]} want {top[i:i + 3].tolist()} (n={len(gd)}/{len(top)})")
    if sc is not None:
        gs = np.array([h[4] for h in got.hits], dtype=np.float32)
        assert np.array_equal(gs.view(np.uint32), sc.view(np.uint32)), f"{ctx}: f32 score bits differ from the restatement"
