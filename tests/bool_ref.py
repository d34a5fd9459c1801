"""The boolean combination rule of a query tree, restated over whole-split arrays, and the scored leaves of
bool_corpora (computed from the corpus arrays, never from the image).

  * bool: a doc matches when it matches every required clause (MUST, FILTER), no MUST_NOT clause, and at least
    `need` SHOULD clauses, where need = minimum_should_match, or 1 when the bool has no required clause (0 then);
  * score: f32(sum of the scored MUST clauses in plan order) + f32(sum of the matching SHOULD clauses in plan order),
    each sum in f32; FILTER and MUST_NOT clauses never score;
  * leaves: a term or phrase scores helpers.bm25_contributions with the plan's f32 weight (scoring_ref); a range,
    exists or match_all scores its boost where it matches; a term set is the union of its terms' postings, unscored.

`evaluate` takes the leaf evaluator as an argument: column_ref uses it with its own leaves."""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np

from quickwit_b200 import ffi, plan as P
import column_ref as CR
import scoring_ref as SR
from helpers import bm25_contributions

MUST, SHOULD, MUST_NOT, FILTER = ffi.OCCUR_MUST, ffi.OCCUR_SHOULD, ffi.OCCUR_MUST_NOT, ffi.OCCUR_FILTER
F32 = np.float32


def evaluate(q, leaf: Callable, n: int) -> Tuple[np.ndarray, np.ndarray]:
    """(match mask, f32 score) of clause q over n docs; `leaf(q)` gives the same pair for a clause that is not a bool
    (its score where it matches, 0 elsewhere)."""
    if q.kind != "bool":
        return leaf(q)
    req = np.ones(n, dtype=bool)
    n_req = 0
    excl = np.zeros(n, dtype=bool)
    cnt = np.zeros(n, dtype=np.int64)
    msum = np.zeros(n, dtype=F32)
    ssum = np.zeros(n, dtype=F32)
    for ch in q.children:
        m, s = evaluate(ch, leaf, n)
        with np.errstate(over="ignore"):   # f32 sums may overflow to +-inf, as the kernel's do
            if ch.occur in (MUST, FILTER):
                req &= m
                n_req += 1
                if ch.occur == MUST:
                    msum = (msum + np.where(m, s, F32(0))).astype(F32)
            elif ch.occur == SHOULD:
                cnt += m
                ssum = (ssum + np.where(m, s, F32(0))).astype(F32)
            else:
                excl |= m
    need = q.msm if q.msm else (1 if n_req == 0 else 0)
    m = req & ~excl & (cnt >= need)
    with np.errstate(over="ignore"):
        return m, np.where(m, (msum + ssum).astype(F32), F32(0)).astype(F32)


class Q:
    """One clause of a bool_corpora plan. kind: bool, term, phrase, term_set, range, exists, all.
    `boost` scales a term's or phrase's BM25 weight (computed from the split's statistics, as the plan carries it), or
    is the score of a range / exists / match_all."""

    def __init__(self, kind: str, occur: int = MUST, field: Optional[str] = None, terms: Sequence[str] = (),
                 col: Optional[str] = None, lo: int = 0, hi: int = 0, children: Sequence["Q"] = (),
                 msm: Optional[int] = None, boost: float = 1.0):
        self.kind, self.occur, self.field, self.terms = kind, occur, field, list(terms)
        self.col, self.lo, self.hi, self.children, self.msm = col, lo, hi, list(children), msm
        self.boost = boost

    def __repr__(self):
        o = "+" if self.occur == MUST else "#" if self.occur == FILTER else "?" if self.occur == SHOULD else "-"
        if self.kind == "bool":
            return f"{o}({' '.join(map(repr, self.children))}{'' if self.msm is None else f' msm={self.msm}'})"
        if self.kind in ("term", "phrase", "term_set"):
            b = "" if self.boost == 1.0 else f"^{self.boost:g}"
            return f"{o}{self.kind[0]}:{self.field}:{'_'.join(self.terms)}{b}"
        if self.kind == "all":
            return f"{o}all^{self.boost:g}"
        return f"{o}{self.kind}:{self.col}[{self.lo:#x},{self.hi:#x}]^{self.boost:g}"


def term(field, t, occur=MUST, boost=1.0):
    return Q("term", occur, field, [t], boost=boost)


def phrase(field, ts, occur=MUST, boost=1.0):
    return Q("phrase", occur, field, ts, boost=boost)


def term_set(field, ts, occur=FILTER):
    return Q("term_set", occur, field, sorted(ts))


def rng(col, lo, hi, occur=FILTER, boost=1.0):
    return Q("range", occur, col=col, lo=lo, hi=hi, boost=boost)


def exists(col, occur=FILTER, boost=1.0):
    return Q("exists", occur, col=col, boost=boost)


def all_(occur=MUST, boost=1.0):
    return Q("all", occur, boost=boost)


def bool_(children, msm=None, occur=MUST):
    return Q("bool", occur, children=children, msm=msm)


# ---- the plan and the leaves over a bool_corpora split -----------------------------------------------------------
def node(sp, q: Q) -> P.Node:
    img = sp.img
    if q.kind == "bool":
        return P.bool_([node(sp, c) for c in q.children], q.msm, q.occur)
    if q.kind == "term":
        return P.term(img, q.field, q.terms[0], q.occur, q.boost)
    if q.kind == "phrase":
        return P.phrase(img, q.field, q.terms, q.occur, q.boost)
    if q.kind == "term_set":
        ords = sorted(o for o in (img.term_ord(q.field, t) for t in q.terms) if o >= 0)
        return P.term_set(img, q.field, ords, q.occur)
    if q.kind == "range":
        return P.range_(img, q.col, q.lo, q.hi, q.occur, q.boost)
    n = P.exists(img, q.col, q.occur) if q.kind == "exists" else P.match_all(q.occur)
    n.boost = q.boost
    return n


def leaf(sp, q: Q) -> Tuple[np.ndarray, np.ndarray]:
    n = sp.n
    m = np.zeros(n, dtype=bool)
    s = np.zeros(n, dtype=F32)
    if q.kind in ("term", "phrase"):
        if any((q.field, t) not in sp.postings for t in q.terms):
            return m, s
        cl = SR.Clause(q.field, q.terms, q.boost)
        docs, tfs = cl.postings(sp)
        w = cl.weight(sp)
        m[docs] = True
        s[docs] = bm25_contributions(tfs, SR.norms(sp, q.field)[docs], w)
        return m, s
    if q.kind == "term_set":
        for t in q.terms:
            if (q.field, t) in sp.postings:
                m[sp.postings[(q.field, t)][0].astype(np.int64)] = True
        return m, s
    if q.kind == "all":
        m[:] = True
    else:
        c = sp.cols.get(q.col)
        if c is not None:
            m = c.has.copy() if q.kind == "exists" else CR.range_mask(c, q.lo, q.hi)
    return m, np.where(m, F32(q.boost), F32(0)).astype(F32)


def eval_split(sp, q: Q) -> Tuple[np.ndarray, np.ndarray]:
    return evaluate(q, lambda x: leaf(sp, x), sp.n)


def plan(sp, q: Q, sort: CR.Sort, K: int, sa=None) -> bytes:
    return P.make_plan(node(sp, q), K, sort.spec(sp), search_after=sa)


def check(got, sp, q: Q, sort: CR.Sort, K: int, sa=None, ctx: str = ""):
    """`got` (a GPU or oracle result) against the restatement: num_hits, (doc, flags, v1, v2) of every hit and, when
    the plan scores (a _score sort key), the f32 score bits of every hit."""
    scoring = any(k == ffi.SORT_SCORE for k, _, _ in sort.keys)
    CR.check(got, sp, q, sort, K, sa, scored=scoring, ctx=ctx, ev=eval_split)


# ---- the lowering's shape of a plan (engine.cu lower_node / lower_plan), for the shared-memory layout and the
# term-slot order --------------------------------------------------------------------------------------------------
class Shape:
    def __init__(self):
        self.n_instr = 0
        self.levels = 0
        self.need_cnt = self.need_msum = self.need_ssum = 0
        self.cols = set()
        self.fn_fields: List[str] = []
        self.slots: List[Q] = []        # TERM instructions in program order (term slot order)
        self.rangeq = False


def _order(q: Q, scored_ctx: bool) -> List[Q]:
    """A bool's children in program order: scored MUST clauses, other required posting clauses, required column
    clauses, SHOULD, MUST_NOT."""
    ch = q.children
    req = [c for c in ch if c.occur in (MUST, FILTER)]
    colpred = lambda c: c.kind in ("range", "exists", "all")
    first = [c for c in req if scored_ctx and c.occur == MUST]
    rest = [c for c in req if not (scored_ctx and c.occur == MUST)]
    return first + [c for c in rest if not colpred(c)] + [c for c in rest if colpred(c)] + \
        [c for c in ch if c.occur == SHOULD] + [c for c in ch if c.occur == MUST_NOT]


def shape(sp, q: Q, scoring: bool, sort: CR.Sort) -> Shape:
    sh = Shape()
    img = sp.img

    def walk(x: Q, level: int, occur: int, scored_ctx: bool):
        scored = scored_ctx and occur in (MUST, SHOULD)
        sh.n_instr += 1
        if x.kind == "bool":
            sh.n_instr += 1
            sh.levels |= 1 << level
            n_req = sum(c.occur in (MUST, FILTER) for c in x.children)
            for c in _order(x, scored):
                if scored and c.occur == MUST:
                    sh.need_msum |= 1 << level
                if scored and c.occur == SHOULD:
                    sh.need_ssum |= 1 << level
                walk(c, level + 1 if c.kind == "bool" else level, c.occur, scored)
            need = x.msm if x.msm else (1 if n_req == 0 else 0)
            if need >= 2:
                sh.need_cnt |= 1 << level
        elif x.kind == "term":
            sh.slots.append(x)
            if scored and img.term_ord(x.field, x.terms[0]) >= 0 and x.field not in sh.fn_fields:
                sh.fn_fields.append(x.field)
        elif x.kind in ("range", "exists"):
            if img.column_ord(x.col) >= 0:
                sh.cols.add(x.col)
            if occur in (MUST, FILTER):
                sh.rangeq = True

    walk(q, 0, MUST, scoring)
    for k, _o, c in sort.keys:
        if k == ffi.SORT_COLUMN and c is not None and img.column_ord(c) >= 0:
            sh.cols.add(c)
    return sh


SIZEOF_DINSTR, SIZEOF_DCOL, SIZEOF_DAGG, SIZEOF_DKEYSPEC = 64, 48, 368, 96
MAX_TERMS, MAX_WBLK, BLK_TAB, HIST_BINS, WARPS = 64, 512, 160, 2048, 16
H100_SMEM_OPTIN = 227 * 1024      # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100
BLOCKS_PER_SM = 2                 # QW_MIN_BLOCKS_PER_SM


def stage_bytes(W: int) -> int:
    return min(max(W, 8192), 24576)


def layout_bytes(W: int, n_levels: int, need_cnt: int, need_msum: int, need_ssum: int, max_instr: int, max_cols: int,
                 n_fn: int, rec_l0: bool, rangeq: bool) -> int:
    """engine.cu make_layout: the k_window arena of a batch, in bytes (no aggregations)."""
    r16 = lambda x: (x + 15) & ~15
    t = r16(32 + 4 * MAX_TERMS + MAX_TERMS) + r16(max(max_instr, 1) * SIZEOF_DINSTR) + r16(max(max_cols, 1) * SIZEOF_DCOL)
    t += SIZEOF_DAGG + SIZEOF_DKEYSPEC
    for lv in range(n_levels):
        t += 3 * r16(W // 8)
        t += r16(W) if (need_cnt >> lv) & 1 else 0
        t += 4 * W * (((need_msum >> lv) & 1) + ((need_ssum >> lv) & 1))
    t += r16(W // 8) + n_fn * W + 16 * MAX_TERMS + 8 * MAX_WBLK + 8 * MAX_TERMS + stage_bytes(W)
    t += 4 * HIST_BINS if rec_l0 else 0
    t += WARPS * (32 + 32 * 4) * 2 if rangeq else 0
    return t


def window_docs(items, optin: int = H100_SMEM_OPTIN) -> int:
    """The k_window window size (engine.cu choose_route) of one call over items (split, Q, Sort, K, sa)."""
    shapes = []
    rec_l0, any_topk = True, False
    for sp, q, sort, K, _sa in items:
        scoring = any(k == ffi.SORT_SCORE for k, _, _ in sort.keys)
        shapes.append(shape(sp, q, scoring, sort))
        if K and sort.keys[0][0] == ffi.SORT_SCORE:
            rec_l0 = False
        any_topk |= K > 0
    nl = max(s.levels.bit_length() for s in shapes)
    args = (nl, _or(s.need_cnt for s in shapes), _or(s.need_msum for s in shapes), _or(s.need_ssum for s in shapes),
            max(s.n_instr + (0 if items[i][1].kind == "bool" else 2) for i, s in enumerate(shapes)),
            max(len(s.cols) for s in shapes), max(len(s.fn_fields) for s in shapes), rec_l0 and any_topk,
            any(s.rangeq for s in shapes))
    W = 32768
    while layout_bytes(W, *args) + 1024 > optin // BLOCKS_PER_SM and W > 1024:
        W //= 2
    return W


def _or(xs):
    out = 0
    for x in xs:
        out |= x
    return out
