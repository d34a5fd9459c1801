"""GPU (seam C) vs CPU oracle on shapes the BASELINE-like corpus never produces.

1. A CLUSTERED split built posting by posting: a term in every doc (0-bit deltas), bursts of consecutive
   docs, a term whose two postings are a whole split apart (wide deltas), tfs above the tf-factor table
   (tf >= 16 divides), a field without fieldnorms / freqs, optional and multi-valued columns. The BM25-union
   pipeline (k_union) meets dense windows that need several slots, windows without postings, tail blocks.
2. Unions with more terms than one slot can stage (clause order across slots) and more than the pipeline
   takes at all (33+ terms -> generic window kernel).
3. hypothesis-driven random bool trees x sort specs x K x aggregations against the oracle.
Everything is bit-exact: doc ids, f32 score bits, sort values, hit counts, bucket counts."""
import random

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings, strategies as st

from quickwit_b200 import ffi, plan as P, splitgen as S
from oracle import oracle as O
from helpers import DOC_ASC, DOC_DESC, SCORE_DESC, assert_same, col_sort, histogram_agg, stats_agg, terms_agg

pytestmark = pytest.mark.gpu

N = 120_000


def _clustered_split(split_id="clustered-0", n=N, seed=5):
    rnd = random.Random(seed)
    b = S._Builder(n)
    lengths = np.array([1 + (i * 7919) % 40 + (300 if i % 1000 == 0 else 0) for i in range(n)], dtype=np.uint32)
    L = ffi.img_lib()
    fn = np.array([L.qwgpu_fieldnorm_to_id(int(x)) for x in lengths], dtype=np.uint8)
    body = b.add_field("body", ffi.FIELD_HAS_FREQS | ffi.FIELD_HAS_FIELDNORMS, ffi.TOK_DEFAULT, fn, int(lengths.sum()))
    tag = b.add_field("tag", 0, ffi.TOK_RAW, None, n)  # record: basic, no fieldnorms

    def add(field, name, docs, tfs=None):
        docs = np.array(sorted(set(docs)), dtype=np.uint32)
        if tfs is None and field == body:
            tfs = np.array([1 + (int(d) * 31) % 3 for d in docs], dtype=np.uint32)
        b.add_term(field, name.encode(), docs, tfs)

    add(body, "every", range(n))                                             # df = 100 %: 0-bit deltas
    add(body, "most", [d for d in range(n) if d % 10 != 3])                 # 90 %
    add(body, "burst", list(range(5_000, 5_700)) + list(range(61_000, 61_130)) + [n - 1])
    add(body, "ends", [0, n - 1])                                            # one block spanning the split
    add(body, "rare", [17, 40_000, 40_001, 99_999])
    add(body, "heavy", range(30_000, 30_400), np.array([1 + (d % 60) for d in range(400)], dtype=np.uint32))  # tf up to 60
    add(body, "third", range(0, n, 3))
    add(body, "half_a", [d for d in range(n) if (d * 2654435761) % 97 < 48])
    add(body, "half_b", [d for d in range(n) if (d * 40503) % 89 < 45])
    for i in range(40):                                                      # many sparse terms (slot overflow, > 32 clauses)
        add(body, f"s{i}", rnd.sample(range(n), 150 + 13 * i))
    # few postings per doc overall, but many contributions on the SAME docs: three dense clauses over one region
    # and five clauses on every 97th doc
    for i in range(3):
        add(body, f"c{i}", range(10_000, 46_000), np.array([1 + ((d + i) % 5) for d in range(36_000)], dtype=np.uint32))
    for i in range(5):
        add(body, f"m{i}", [d for d in range(n) if d % 97 == 5], np.array([1 + ((d * (i + 3)) % 7) for d in range(len(range(5, n, 97)))], dtype=np.uint32))
    add(tag, "A", [d for d in range(n) if d % 4 == 0])
    add(tag, "B", [d for d in range(n) if d % 4 == 1])
    ts = np.array([S.i64_to_u64((1_700_000_000 + d // 3) * 1_000_000_000) for d in range(n)], dtype=np.uint64)
    b.add_column("timestamp", ffi.COL_DATETIME, ffi.CARD_FULL, ts, None)
    b.add_column("code", ffi.COL_U64, ffi.CARD_FULL, np.array([(d * 7) % 5 for d in range(n)], dtype=np.uint64), None)
    opt_docs = np.array([d for d in range(n) if d % 5 != 0], dtype=np.uint32)
    b.add_column("opt", ffi.COL_I64, ffi.CARD_OPTIONAL,
                 np.array([S.i64_to_u64(((int(d) * 37) % 2001) - 1000) for d in opt_docs], dtype=np.uint64), opt_docs)
    return b.finish(split_id)


@pytest.fixture(scope="module")
def clustered(gpu_ctx):
    img = _clustered_split()
    gpu_ctx.register_split(img)
    yield img
    gpu_ctx.unregister_split(img.split_id)


def run_both(sctx, img, plan, **kw):
    got = sctx.split_search([img.split_id], [plan])[0]
    want = O.split_search(img, plan)
    assert_same(got, want, **kw)
    return got, want


def B(img, name, occur=ffi.OCCUR_SHOULD, boost=1.0, field="body"):
    return P.term(img, field, name, occur=occur, boost=boost)


def test_clustered_unions(gpu_ctx, clustered):
    img = clustered
    cases = {
        "dense + sparse": ["every", "most", "burst", "ends", "rare"],
        "sparse first, dense last": ["rare", "ends", "burst", "third", "every"],
        "tf above the factor table": ["heavy", "third", "rare"],
        "single dense": ["every"],
        "single two-posting term": ["ends"],
        "two halves": ["half_a", "half_b", "most"],
    }
    for name, terms in cases.items():
        for k in (1, 10, 1000, 4096):
            root = P.bool_([B(img, t) for t in terms])
            got, _ = run_both(gpu_ctx, img, P.make_plan(root, k, SCORE_DESC), ctx=f"{name} k={k}")
            assert len(got.hits) == min(k, got.num_hits)
    # boosts, an absent term, a field without freqs / fieldnorms in the same union
    root = P.bool_([B(img, "third", boost=3.0), B(img, "nope"), B(img, "A", field="tag"), B(img, "burst", boost=0.25)])
    run_both(gpu_ctx, img, P.make_plan(root, 200, SCORE_DESC), ctx="mixed fields")
    # second sort key on top of the score
    run_both(gpu_ctx, img, P.make_plan(P.bool_([B(img, "third"), B(img, "burst")]), 300,
                                       [(ffi.SORT_SCORE, ffi.ORDER_DESC, ffi.ABSENT), col_sort(img, "timestamp", ffi.ORDER_ASC)]), ctx="score then ts")


def test_many_contributions_per_doc(gpu_ctx, clustered):
    """Unions with few postings per doc overall but many contributions on the SAME docs (five clauses on every
    97th doc, three dense clauses over one region): every f32 score equals the oracle's clause-order sum bit
    for bit."""
    img = clustered
    fold = ["m3", "m0", "rare", "m4", "m1", "m2", "burst"]          # 5 contributions on every 97th doc
    for k in (10, 2000):
        got, _ = run_both(gpu_ctx, img, P.make_plan(P.bool_([B(img, t, boost=1.0 + 0.37 * i) for i, t in enumerate(fold)]), k, SCORE_DESC), ctx=f"fold k={k}")
        # 120 000 docs are too few windows to sample: the exact radix descent runs from the start (the sampled
        # threshold on these shapes is covered by test_gpu_topk_threshold.py)
        assert got.sample_stride == 0 and got.exact_fallbacks == 0 and got.radix_passes >= 1
    dense = ["c0", "ends", "c1", "c2"]                               # 3 contributions on 36 000 consecutive docs
    run_both(gpu_ctx, img, P.make_plan(P.bool_([B(img, t, boost=1.0 + 0.21 * i) for i, t in enumerate(dense)]), 100, SCORE_DESC), ctx="dense")
    mixed = ["c0", "m0", "c1", "m1", "s3", "m2"]                     # two planes + list + sparse clauses
    run_both(gpu_ctx, img, P.make_plan(P.bool_([B(img, t) for t in mixed]), 500, SCORE_DESC), ctx="mixed")


def test_many_clause_unions(gpu_ctx, clustered):
    img = clustered
    for n_terms, extra in [(12, []), (31, ["most"]), (32, []), (33, []), (40, ["every", "third"])]:
        terms = [f"s{i}" for i in range(min(n_terms, 40))] + extra
        root = P.bool_([B(img, t) for t in terms])
        run_both(gpu_ctx, img, P.make_plan(root, 500, SCORE_DESC), ctx=f"{len(terms)} clauses")


_TERMS = ["every", "most", "burst", "ends", "rare", "heavy", "third", "half_a", "half_b", "s0", "s7", "s39", "nope"]
_OCC = [ffi.OCCUR_MUST, ffi.OCCUR_SHOULD, ffi.OCCUR_SHOULD, ffi.OCCUR_MUST_NOT, ffi.OCCUR_FILTER]


@st.composite
def _leaf(draw, img_cols):
    kind = draw(st.sampled_from(["term", "term", "term", "range", "exists", "all"]))
    occ = draw(st.sampled_from(_OCC))
    if kind == "term":
        return ("term", draw(st.sampled_from(_TERMS)), occ, draw(st.sampled_from([1.0, 1.0, 2.0, 0.5])))
    if kind == "range":
        col = draw(st.sampled_from(["timestamp", "code", "opt", "missing_col"]))
        return ("range", col, occ, draw(st.integers(0, 1000)), draw(st.integers(0, 1000)))
    if kind == "exists":
        return ("exists", draw(st.sampled_from(["opt", "code", "missing_col"])), occ)
    return ("all", occ)


@st.composite
def _tree(draw, depth=0):
    n = draw(st.integers(1, 4))
    kids = []
    for _ in range(n):
        if depth < 2 and draw(st.integers(0, 4)) == 0:
            kids.append(("bool", draw(_tree(depth + 1)), draw(st.sampled_from(_OCC)), draw(st.sampled_from([None, None, 1, 2]))))
        else:
            kids.append(draw(_leaf(None)))
    return kids


def _build(img, kids, msm=None, occur=ffi.OCCUR_MUST):
    nodes = []
    for k in kids:
        if k[0] == "term":
            nodes.append(P.term(img, "body", k[1], occur=k[2], boost=k[3]))
        elif k[0] == "range":
            c = img.column_ord(k[1])
            if c < 0:
                nodes.append(P.Node(ffi.NODE_RANGE, k[2], column=ffi.ABSENT))
            else:
                col = img.columns()[c]
                span = col.max_value - col.min_value
                lo, hi = sorted((col.min_value + span * k[3] // 1000, col.min_value + span * k[4] // 1000))
                nodes.append(P.range_(img, k[1], lo, hi, occur=k[2]))
        elif k[0] == "exists":
            nodes.append(P.exists(img, k[1], occur=k[2]))
        elif k[0] == "all":
            nodes.append(P.match_all(occur=k[1]))
        else:
            nodes.append(_build(img, k[1], msm=k[3], occur=k[2]))
    return P.bool_(nodes, min_should_match=msm, occur=occur)


_SORTS = st.sampled_from(["score", "score_asc", "doc", "doc_asc", "ts", "ts_asc", "code_ts", "opt_desc", "opt_asc_score", "missing"])


def _sort(img, name):
    return {
        "score": SCORE_DESC, "score_asc": [(ffi.SORT_SCORE, ffi.ORDER_ASC, ffi.ABSENT)], "doc": DOC_DESC, "doc_asc": DOC_ASC,
        "ts": [col_sort(img, "timestamp", ffi.ORDER_DESC)], "ts_asc": [col_sort(img, "timestamp", ffi.ORDER_ASC)],
        "code_ts": [col_sort(img, "code", ffi.ORDER_ASC), col_sort(img, "timestamp", ffi.ORDER_DESC)],
        "opt_desc": [col_sort(img, "opt", ffi.ORDER_DESC)],
        "opt_asc_score": [col_sort(img, "opt", ffi.ORDER_ASC), (ffi.SORT_SCORE, ffi.ORDER_DESC, ffi.ABSENT)],
        "missing": [col_sort(img, "missing_col", ffi.ORDER_DESC)],
    }[name]


@settings(max_examples=70, deadline=None, derandomize=True, suppress_health_check=list(HealthCheck))
@given(kids=_tree(), msm=st.sampled_from([None, None, 1, 2]), sort=_SORTS, k=st.sampled_from([0, 1, 7, 100, 1000]),
       with_aggs=st.integers(0, 3))
def test_random_plans_against_the_oracle(gpu_ctx, clustered, kids, msm, sort, k, with_aggs):
    img = clustered
    root = _build(img, kids, msm=msm)
    aggs = []
    if with_aggs == 1:
        aggs = [terms_agg(img, "code"), histogram_agg(img, "timestamp", 3600e9)]
    elif with_aggs == 2:
        aggs = [terms_agg(img, "code", children=[stats_agg(img, "timestamp")]), stats_agg(img, "opt")]
    plan = P.make_plan(root, k, _sort(img, sort), aggs=aggs)
    run_both(gpu_ctx, img, plan, ctx=f"kids={kids} msm={msm} sort={sort} k={k} aggs={with_aggs}")


# ---- phrases ------------------------------------------------------------------------------------------------------
_VOCAB = ["alpha", "beta", "gamma", "delta", "eps", "zeta", "eta", "theta"]


@pytest.fixture(scope="module")
def phrase_split(gpu_ctx):
    """20 000 docs of 3..40 random words over 8 words (every word in most docs, every 2-word phrase frequent, long
    phrases rare), a multi-valued field, many posting blocks per term."""
    rnd = random.Random(11)
    docs = []
    for i in range(20_000):
        n = 3 + (i * 37) % 38
        doc = {"body": " ".join(rnd.choice(_VOCAB) for _ in range(n)), "n": i % 50}
        if i % 3 == 0:
            doc["tags"] = [" ".join(rnd.choice(_VOCAB[:4]) for _ in range(1 + i % 3)) for _ in range(1 + i % 4)]
        if i % 1000 == 0:
            doc["body"] += " " + " ".join(["alpha beta"] * 20)   # phrase_count above the tf-factor table
        docs.append(doc)
    mapping = {"field_mappings": [{"name": "body", "type": "text", "record": "position", "fieldnorms": True},
                                  {"name": "tags", "type": "text", "record": "position"},
                                  {"name": "n", "type": "u64", "fast": True}]}
    img = S.build_split(docs, mapping, "phrases-0")
    gpu_ctx.register_split(img)
    yield img
    gpu_ctx.unregister_split(img.split_id)


def test_phrases_against_the_oracle(gpu_ctx, phrase_split):
    img = phrase_split
    rnd = random.Random(3)
    cases = [["alpha", "beta"], ["beta", "alpha"], ["alpha", "alpha"], ["alpha", "beta", "gamma"], ["eta", "eta", "eta"],
             ["alpha", "beta", "gamma", "delta"], ["theta", "zeta", "eta", "eps", "delta", "gamma", "beta", "alpha"]]
    cases += [[rnd.choice(_VOCAB) for _ in range(rnd.randint(2, 5))] for _ in range(12)]
    n_hits = []
    for terms in cases:
        for k, sort in ((10, SCORE_DESC), (300, DOC_ASC), (0, DOC_DESC)):
            got, _ = run_both(gpu_ctx, img, P.make_plan(P.phrase(img, "body", terms), k, sort), ctx=f"phrase {terms} k={k}")
        n_hits.append(got.num_hits)
    assert max(n_hits) > 5000 and 0 < min(x for x in n_hits if x) < 200      # frequent and rare phrases both occurred
    # multi-valued field without fieldnorms
    for terms in (["alpha", "beta"], ["gamma", "delta", "alpha"], ["beta", "beta"]):
        run_both(gpu_ctx, img, P.make_plan(P.phrase(img, "tags", terms), 50, SCORE_DESC), ctx=f"tags {terms}")
    # phrases as clauses: must + should + must_not, two phrases in a union, a range filter, an aggregation
    ph = lambda terms, occ, boost=1.0, field="body": P.phrase(img, field, terms, occur=occ, boost=boost)
    t = lambda name, occ: P.term(img, "body", name, occur=occ)
    plans = [
        P.bool_([ph(["alpha", "beta"], ffi.OCCUR_MUST), t("gamma", ffi.OCCUR_SHOULD), ph(["delta", "delta"], ffi.OCCUR_MUST_NOT)]),
        P.bool_([ph(["alpha", "beta"], ffi.OCCUR_SHOULD, 2.0), ph(["gamma", "delta"], ffi.OCCUR_SHOULD), t("eta", ffi.OCCUR_SHOULD)]),
        P.bool_([ph(["alpha", "beta"], ffi.OCCUR_SHOULD), ph(["gamma", "delta"], ffi.OCCUR_SHOULD), ph(["alpha", "gamma"], ffi.OCCUR_SHOULD, field="tags")],
                min_should_match=2),
        P.bool_([ph(["zeta", "eta"], ffi.OCCUR_MUST), P.range_(img, "n", 10, 30, occur=ffi.OCCUR_FILTER)]),
        P.bool_([t("alpha", ffi.OCCUR_MUST), ph(["beta", "gamma", "delta"], ffi.OCCUR_FILTER)]),
    ]
    for i, root in enumerate(plans):
        for k, sort in ((25, SCORE_DESC), (1000, [col_sort(img, "n", ffi.ORDER_ASC), (ffi.SORT_SCORE, ffi.ORDER_DESC, ffi.ABSENT)])):
            run_both(gpu_ctx, img, P.make_plan(root, k, sort), ctx=f"phrase plan {i} k={k}")
    run_both(gpu_ctx, img, P.make_plan(ph(["alpha", "beta"], ffi.OCCUR_MUST), 0, DOC_DESC, aggs=[terms_agg(img, "n")]), ctx="phrase + terms agg")


@pytest.mark.gpu
def test_phrases_over_the_synthetic_positions_field(gpu_ctx):
    """The bench corpus' optional `msg` field (positions, Zipf vocabulary): frequent 2-word and rarer 3-word
    phrases at a size where every term spans thousands of posting blocks — the BASELINE config 5 queries."""
    img = S.synth_split(400_000, 7, [0.2, 0.05], split_id="synth-msg-7", msg_vocab=64)
    gpu_ctx.register_split(img)
    try:
        counts = []
        for terms in (["w1", "w2"], ["w0", "w3", "w1"], ["w40", "w50"], ["w5", "w5"]):
            for k, sort in ((10, SCORE_DESC), (200, DOC_DESC)):
                got, _ = run_both(gpu_ctx, img, P.make_plan(P.phrase(img, "msg", terms), k, sort), ctx=f"msg phrase {terms} k={k}")
            counts.append(got.num_hits)
        assert counts[0] > 5000 and counts[1] > 100 and counts[2] < counts[0]
        # a phrase next to a scored body term and a timestamp sort
        root = P.bool_([P.phrase(img, "msg", ["w1", "w2"], occur=ffi.OCCUR_MUST), P.term(img, "body", "t0", occur=ffi.OCCUR_SHOULD)])
        run_both(gpu_ctx, img, P.make_plan(root, 100, SCORE_DESC), ctx="msg phrase + body term")
        run_both(gpu_ctx, img, P.make_plan(root, 100, [col_sort(img, "timestamp", ffi.ORDER_DESC)]), ctx="msg phrase by timestamp")
    finally:
        gpu_ctx.unregister_split(img.split_id)
