"""The `_score` bucket-edge corpora, checked without a GPU: every planted doc realises the edge its class claims
(digit and ulp distance restated from its lengths through the fieldnorm table), the restated key orders docs as the brute force
does, and the CPU oracle agrees with the brute force on every plan of tests/test_gpu_score_edges.py."""
import numpy as np
import pytest

from quickwit_b200 import ffi, plan as P
from oracle import oracle as O
from helpers import SCORE_DESC
import score_edges_ref as R

SCORE_ASC = [(ffi.SORT_SCORE, ffi.ORDER_ASC, ffi.ABSENT)]


@pytest.fixture(scope="module")
def corpus():
    return R.EdgeCorpus(200_000, "edges-host")


@pytest.mark.parametrize("t", list(R.EDGE_TERMS) + ["asc"])
def test_planted_docs_sit_on_their_edges(corpus, t):
    c = corpus
    scale = c.scale(c.clauses(t))
    s = c.scores(c.clauses(t))
    l = c.l[t]
    pa, ne, pb, nm = R.ASC if t == "asc" else R.EDGE_TERMS[t]
    cls = c.planted[t]
    x = {k: R.fmul(s[v], scale) for k, v in cls.items()}
    u = {k: R.ulps_from(v, l) for k, v in x.items()}
    # exactly on l, and rounded up to it: a truncating multiply would put the tie one bucket lower
    assert len(cls["exact"]) == ne and (u["exact"] == 0).all()
    assert R.rounds_up(s[cls["exact"]], scale).all()
    assert len(np.unique(s[cls["exact"]].view(np.uint32))) == 1, "one tie, one score"
    assert (R.lin(s[cls["exact"]], scale) == l).all()
    # 1..8 ulps above l: bucket l, inside the band a x1.000001 bound would drop; every ulp realised
    if len(cls["above"]):
        assert set(u["above"].tolist()) == set(range(1, 1 + min(R.BAND, len(cls["above"]))))
        assert (R.lin(s[cls["above"]], scale) == l).all()
        if t != "asc":   # (the ASC plan never takes these bounds)
            mutated = np.float32(np.float32(np.float32(l) / scale) * np.float32(1.000001))
            assert (s[cls["above"]] < mutated).all() and (s[cls["exact"]] < mutated).all()
    # 1..8 ulps below l: bucket l - 1
    assert set(u["below"].tolist()) == set(range(-R.BAND, 0))
    assert (R.lin(s[cls["below"]], scale) == l - 1).all()
    # the bounds of both routes keep every doc of bucket l, and the band below them holds only bucket l - 1
    for k in ("above", "exact"):
        assert R.passes_union(s[cls[k]], l, scale).all() and R.passes_window(s[cls[k]], l, scale).all()
    lo = R.s_lo_union(l, scale)
    assert R.lin(lo, scale) == l - 1 and R.lin(np.nextafter(lo, np.float32(np.inf)), scale) <= l
    if nm:
        want = l if t == "asc" else l - 1
        assert (R.lin(s[cls["mass"]], scale) == want).all()
        assert (np.abs(u["mass"]) > R.BAND).all()


def test_top_reaches_the_clamp(corpus):
    c = corpus
    w = c.weight("top")
    scale = R.score_scale([w])
    s = c.scores([("top", 1.0)])
    mx = c.planted["top"]["max"]
    assert (s[mx] == w).all(), "tf 2^32 - 1 scores the whole weight: score == score_max"
    x = R.fmul(s[mx], scale)
    assert (x >= 1023).all() and (R.lin(s[mx], scale) == 1023).all()
    near = c.planted["top"]["near"]
    u = R.ulps_from(R.fmul(s[near], scale), 1023)
    assert (u == 0).any() and (u < 0).any() and (u > 0).any()
    # x = 1024: without the clamp the digit would be 1024 | 1024 = 1024, bucket 0
    assert (R.fmul(s[mx], scale) == 1024).all()


def test_union_reaches_the_clamp(corpus):
    """`ca OR cb` at both clauses' tf 2^32 - 1 scores score_max (the f32 sum of the weights in clause order) at x = 1024;
    other docs sit on both sides of x = 1023; the tie of ca alone sits in one bucket far below."""
    c = corpus
    cl = c.clamp_clauses()
    scale = c.scale(cl)
    s = c.scores(cl)
    smax = np.float32(c.weight(*cl[0]) + c.weight(*cl[1]))
    assert scale == R.score_scale([c.weight(*cl[0]), c.weight(*cl[1])])
    p = c.planted["ca"]
    assert (s[p["max"]] == smax).all() and (R.fmul(s[p["max"]], scale) == 1024).all()
    assert (R.lin(s[p["max"]], scale) == 1023).all() and (R.digit(s[p["max"]], scale) == 2047).all()
    u = R.ulps_from(R.fmul(s[p["near"]], scale), 1023)
    assert (u == 0).any() and (u < 0).any() and (u > 0).any()
    assert len(np.unique(s[p["mass"]].view(np.uint32))) == 1 and R.lin(s[p["mass"]][:1], scale)[0] < 1000
    assert len(p["mass"]) > 8192 - len(p["max"]) - len(p["near"]), "a threshold in the tie's bucket overflows"


def test_key_orders_as_the_brute_force(corpus):
    c = corpus
    for t, desc in [("e10", True), ("e1000", True), ("asc", False)]:
        s = c.scores(c.clauses(t))
        m = c.tf[t] > 0
        order = R.brute_order(s, m, desc)
        k = R.keys(s[order], order, c.scale(c.clauses(t)), int(c.n - 1).bit_length(), desc)
        assert k.dtype == np.uint64 and (k[:-1] > k[1:]).all(), "keys strictly decrease in rank order"


def _plans(c):
    """Every plan of the GPU module, with its brute force: (plan, matched mask, scores, desc, skip)."""
    def clauses(cl, must_not=()):
        kids = [P.term(c.img, "body", t, occur=ffi.OCCUR_SHOULD, boost=b) for t, b in cl]
        kids += [P.term(c.img, "body", t, occur=ffi.OCCUR_MUST_NOT) for t in must_not]
        return P.bool_(kids)

    def mask(cl, must_not=()):
        m = np.zeros(c.n, dtype=bool)
        for t, _ in cl:
            m |= c.tf[t] > 0
        for t in must_not:
            m &= c.tf[t] == 0
        return m

    out = []
    for t, K in (("e1", 1), ("e10", 10), ("e1000", 1000), ("e4096", 4096), ("e4096", 4097)):
        for mn in ((), ("x",)):
            out.append((P.make_plan(clauses(c.clauses(t), mn), K, SCORE_DESC), mask(c.clauses(t), mn), c.scores(c.clauses(t)), True))
    for K in (10, 1000):
        out.append((P.make_plan(clauses(c.clauses("asc")), K, SCORE_ASC), mask(c.clauses("asc")), c.scores(c.clauses("asc")), False))
    for K in (10, 1000):
        out.append((P.make_plan(clauses(c.clamp_clauses()), K, SCORE_DESC), mask(c.clamp_clauses()), c.scores(c.clamp_clauses()), True))
    for K in (10, 50):
        root = P.bool_([P.term(c.img, "body", "top"), P.range_(c.img, "f", 0, 0)])
        out.append((P.make_plan(root, K, SCORE_DESC), (c.tf["top"] > 0) & (c.f == 0), c.scores([("top", 1.0)]), True))
    cl = [("tune_e1", 1000.0), ("g", 1.0)]
    for mn in ((), ("x",)):
        out.append((P.make_plan(clauses(cl, mn), 1000, SCORE_DESC), mask(cl, mn), c.scores(cl), True))
    return out


def test_oracle_agrees_with_the_brute_force(corpus):
    c = corpus
    for i, (pl, m, s, desc) in enumerate(_plans(c)):
        want = R.brute_order(s, m, desc)
        got = O.split_search(c.img, pl)
        K = len(got.hits)
        assert got.num_hits == int(m.sum()), i
        assert [h[0] for h in got.hits] == want[:K].tolist(), f"plan {i}"
        gs = np.array([h[4] for h in got.hits], dtype=np.float32).view(np.uint32)
        assert np.array_equal(gs, s[want[:K]].view(np.uint32)), f"plan {i}"
