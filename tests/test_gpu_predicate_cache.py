"""The predicate cache on the GPU (QW_NODE_CACHE, DESIGN.md §4.9). Every plan runs three times: on a context with the
cache disabled, then twice on a context with it enabled (a miss that fills the entry, then a hit that reads it). The
three results (num_hits, hits with their sort values and f32 score bits, aggregation cells) must be identical, equal
to the oracle's for the plan with its CACHE nodes replaced by their children, and to the brute force restatement of
the corpus arrays; QWGPU_KERNEL_PREDICATE_FILL is set on the miss only, and the cache counters move by the expected
misses, fills and hits."""
import json
import threading

import numpy as np
import pytest

from quickwit_b200 import ffi, plan as P, proto
from quickwit_b200.service import SearcherContext
from quickwit_b200 import splitgen as S
from helpers import assert_same, terms_agg
from regex_ref import oracle_search
import bool_corpora as BC
import bool_ref as B
import column_corpora as CC
import column_ref as CR
import test_bool_limits_host as H
from test_predicate_cache_host import DM, parse, strip

pytestmark = pytest.mark.gpu

MUST, SHOULD, MUST_NOT, FILTER = B.MUST, B.SHOULD, B.MUST_NOT, B.FILTER
body, title, tag, ph, ts, rng, bl = H.body, H.title, H.tag, H.ph, H.ts, H.rng, H.bl
BUDGET = 1 << 30


def C(q):
    """q, read through the predicate cache"""
    q.cached = True
    return q


def to_node(sp, q, conv):
    n = P.bool_([to_node(sp, c, conv) for c in q.children], q.msm, q.occur) if q.kind == "bool" else conv(sp, q)
    return P.cache(n) if getattr(q, "cached", False) else n


def plan_of(sp, q, sort, K, sa=None, aggs=()):
    conv = B.node if isinstance(sp, BC.BoolSplit) else CR.node
    return P.make_plan(to_node(sp, q, conv), K, sort.spec(sp), aggs=aggs, search_after=sa)


def brute(got, sp, q, sort, K, sa, ctx):
    if isinstance(sp, BC.BoolSplit):
        B.check(got, sp, q, sort, K, sa, ctx=ctx)
    else:
        CR.check(got, sp, q, sort, K, sa, ctx=ctx)


def key(r):
    return (r.num_hits, [tuple(h[:4]) + (np.float32(h[4]).view(np.uint32),) for h in r.hits], r.cells, sorted(r.entries))


@pytest.fixture(scope="module")
def corpus():
    return {"bool": BC.small_split(), "bool-main": BC.main_split(), "col": CC.main_split(),
            **{f"col-{n}": CC.small_split(n) for n in (1, 1024, 2049)}}


@pytest.fixture(scope="module")
def ctxs(gpu_ctx, corpus):
    pc = SearcherContext(0)
    pc.set_predicate_cache_budget(BUDGET)
    for sp in corpus.values():
        gpu_ctx.register_split(sp.img)
        pc.register_split(sp.img)
    yield gpu_ctx, pc
    for sp in corpus.values():
        gpu_ctx.unregister_split(sp.split_id)
    pc.close()


def entries_read(plan: bytes) -> int:
    """The CACHE nodes of an unscored plan that read an entry: the outermost ones, except those over ALL / NONE (a
    phrase or term absent from a split may compile to NONE)."""
    _, nodes = parse(plan)
    def walk(i):
        n = nodes[i]
        if n.kind == ffi.NODE_CACHE and nodes[n.first_child].kind not in (ffi.NODE_ALL, ffi.NODE_NONE):
            return 1
        if n.kind in (ffi.NODE_BOOL, ffi.NODE_CACHE):
            return sum(walk(n.first_child + k) for k in range(n.num_children))
        return 0
    return walk(0)


def three(ctxs, items, label, fills=True):
    """items: (split, q, sort, K, search_after, aggs). Runs the batch disabled / miss / hit and checks them."""
    off, on = ctxs
    plans = [plan_of(sp, q, sort, K, sa, aggs) for sp, q, sort, K, sa, aggs in items]
    ids = [it[0].split_id for it in items]
    n_cached = sum(entries_read(pl) for pl in plans)
    on.set_predicate_cache_budget(0)  # (every case starts cold: another case may have cached the same subtree)
    on.set_predicate_cache_budget(BUDGET)
    i0 = on.predicate_cache_info()
    r_off = off.split_search(ids, plans)
    r_miss = on.split_search(ids, plans)
    i1 = on.predicate_cache_info()
    r_hit = on.split_search(ids, plans)
    i2 = on.predicate_cache_info()
    for k, (it, pl) in enumerate(zip(items, plans)):
        sp, q, sort, K, sa, aggs = it
        tag_ = f"{label} {sp.split_id} {q!r} K={K}"
        assert key(r_off[k]) == key(r_miss[k]) == key(r_hit[k]), tag_
        want = oracle_search(sp.img, strip(pl))
        assert_same(r_hit[k], want, ctx=tag_)
        if not aggs:
            brute(r_hit[k], sp, q, sort, K, sa, tag_)
    assert not r_off[0].kernel_mask & ffi.KERNEL_PREDICATE_FILL, label
    assert bool(r_miss[0].kernel_mask & ffi.KERNEL_PREDICATE_FILL) == (fills and n_cached > 0), (label, hex(r_miss[0].kernel_mask))
    assert not r_hit[0].kernel_mask & ffi.KERNEL_PREDICATE_FILL, label
    if fills:
        assert i1["misses"] - i0["misses"] == n_cached and i1["fills"] - i0["fills"] == n_cached, (label, i0, i1)
        assert i2["hits"] - i1["hits"] == n_cached and i2["misses"] == i1["misses"], (label, i1, i2)
    return r_off, r_miss, r_hit


BY_U = H.BY_U
BY_I = H.BY_I
DOC = H.DOC_DESC


def level3_cached():
    t = H.deep_tree(False)
    l1 = t.children[0]
    l2a = l1.children[0]
    C(l2a.children[1])  # l3a: a level-3 bool
    return t


def position_cases(sp):
    f = lambda m: bl([tag("a0"), C(body("m01", SHOULD)), body("m02", SHOULD), C(ph("title", ["pa", "pb"], SHOULD))], msm=m)
    return [
        ("root", C(bl([body("m00"), body("m01", SHOULD), rng("c00", 50, 950, FILTER)]))),
        ("must", bl([C(body("m00")), body("m02", SHOULD), tag("a0")])),
        ("filter", bl([body("m00"), C(bl([title("tt00"), body("m03", SHOULD)], occur=FILTER))])),
        *[(f"should msm={m}", f(m)) for m in (None, 0, 1, 2, 3, 4)],
        ("must_not", bl([body("dense"), C(body("s00", MUST_NOT))])),
        ("level 3", level3_cached()),
        ("phrase", bl([tag("a0"), C(ph("title", ["pa", "pb"], FILTER))])),
        # a phrase of more than QW_MAX_PHRASE_TERMS tokens: the fill runs k_phrase_long
        ("long phrase", bl([body("m00", SHOULD), tag("a0", SHOULD), C(ph("title", ["pa", "pb"] * 4 + ["pa"], FILTER))])),
        ("term set", bl([body("m00"), C(ts("title", ["tt01", "tt02", "tt03"], FILTER))])),
        ("range", bl([body("m00", SHOULD), body("m01", SHOULD), C(rng("c01", 0, 600, FILTER))])),
        ("nested", bl([body("m00"), C(bl([C(body("m03")), title("tt00", SHOULD)], occur=FILTER))])),
    ]


@pytest.mark.parametrize("split", ["bool", "bool-main"])
def test_clause_positions(ctxs, corpus, split):
    sp = corpus[split]
    cases = position_cases(sp)
    sorts = ((BY_U, 10), (DOC, 0), (BY_I, 4096))
    if split == "bool-main":  # (528 385 docs: the oracle and the brute force take seconds per plan)
        cases, sorts = cases[:3] + cases[-5:], sorts[:1]
    for label, q in cases:
        for sort, K in sorts:
            three(ctxs, [(sp, q, sort, K, None, ())], f"{label} K={K}")
        # search_after: the page after the first ten hits
        first = ctxs[0].split_search([sp.split_id], [plan_of(sp, q, BY_U, 10)])[0]
        if first.hits:
            sa = CR.after(first.hits[-1])
            three(ctxs, [(sp, q, BY_U, 10, sa, ())], f"{label} search_after")


def test_aggregations(ctxs, corpus):
    sp = corpus["bool"]
    q = bl([C(body("m00")), body("m02", SHOULD)])
    three(ctxs, [(sp, q, BY_U, 10, None, (terms_agg(sp.img, "c00"),))], "terms agg")


@pytest.mark.parametrize("n", [1, 1024, 2049, None])
def test_bitmap_edges(ctxs, corpus, n):
    sp = corpus["col" if n is None else f"col-{n}"]
    hi = int(np.median(sp.cols["w10"].vals))
    qs = [CR.bool_([CR.term("d30", SHOULD), CR.term("all", SHOULD), C(CR.rng("w10", 0, hi))]),
          C(CR.bool_([CR.exists("o10"), CR.term("d30", MUST_NOT)])),
          CR.bool_([CR.term("all"), C(CR.term("d30", MUST_NOT))])]
    for q in qs:
        for sort, K in ((CR.col_sort("w10", ffi.ORDER_DESC), 10), (DOC, 0), (CR.col_sort("w3", ffi.ORDER_ASC), 4096)):
            three(ctxs, [(sp, q, sort, K, None, ())], f"edges n={sp.num_docs}")


def test_mixed_batch(ctxs, corpus):
    """A batch over every split: the splits the last call filled hit, the new one misses."""
    qa = lambda: bl([C(body("m04")), body("m05", SHOULD)])
    qc = lambda: CR.bool_([CR.term("all"), C(CR.term("d30", MUST_NOT))])
    bool_items = [(corpus["bool"], qa(), BY_U, 100, None, ())]
    three(ctxs, bool_items, "mixed warm-up")
    items = bool_items + [(corpus[k], qc(), DOC, 100, None, ()) for k in ("col", "col-1", "col-1024", "col-2049")]
    off, on = ctxs
    plans = [plan_of(sp, q, s, K) for sp, q, s, K, _, _ in items]
    ids = [it[0].split_id for it in items]
    i0 = on.predicate_cache_info()
    got = on.split_search(ids, plans)
    i1 = on.predicate_cache_info()
    assert got[0].kernel_mask & ffi.KERNEL_PREDICATE_FILL
    assert i1["hits"] - i0["hits"] >= 1 and i1["fills"] - i0["fills"] == 4, (i0, i1)
    for g, w in zip(got, off.split_search(ids, plans)):
        assert key(g) == key(w)


def test_route_rule(ctxs, corpus):
    sp = corpus["bool"]
    # a scored CACHE: lowered as its child, nothing is filled
    q = bl([C(body("m00")), body("m02", SHOULD)])
    r = three(ctxs, [(sp, q, H.SC_DESC, 100, None, ())], "scored", fills=False)
    assert all(not x[0].kernel_mask & ffi.KERNEL_PREDICATE_FILL for x in r)
    # the k_driver shape (term + range filter): the stripped plan keeps k_driver, nothing is filled
    q = bl([body("m00"), C(rng("c01", 0, 600, FILTER))])
    r = three(ctxs, [(sp, q, BY_U, 100, None, ())], "driver", fills=False)
    for x in r:
        assert x[0].kernel_mask & ffi.KERNEL_DRIVER and not x[0].kernel_mask & ffi.KERNEL_PREDICATE_FILL, hex(x[0].kernel_mask)


def test_budget(corpus):
    """LRU eviction across splits, a budget below one entry, and budget 0."""
    ctx = SearcherContext(0)
    try:
        sps = [corpus["col"], corpus["col-2049"], corpus["col-1024"]]
        for sp in sps:
            ctx.register_split(sp.img)
        ref = SearcherContext(0)
        for sp in sps:
            ref.register_split(sp.img)
        entry = (corpus["col"].num_docs + 31) // 32 * 4
        ctx.set_predicate_cache_budget(entry + 2 * 300)  # the big split's entry and two small ones, not two big ones
        # (neither is k_driver's shape, which never reads the cache: test_route_rule)
        qs = [C(CR.bool_([CR.term("d30", SHOULD), CR.term("all", SHOULD), CR.exists("o10")])),
              C(CR.bool_([CR.term("all"), CR.term("d30", MUST_NOT)]))]
        for round_ in range(2):
            for q in qs:
                for sp in sps:
                    pl = plan_of(sp, q, DOC, 50)
                    assert key(ctx.split_search([sp.split_id], [pl])[0]) == key(ref.split_search([sp.split_id], [pl])[0])
        info = ctx.predicate_cache_info()
        assert info["evictions"] > 0 and info["used_bytes"] <= info["budget_bytes"], info
        # below one entry of the big split: it never caches (the small ones still do)
        ctx.set_predicate_cache_budget(entry - 4)
        f0 = ctx.predicate_cache_info()["fills"]
        sp = corpus["col"]
        pl = plan_of(sp, C(CR.bool_([CR.term("q128", SHOULD), CR.term("d30", SHOULD), CR.exists("o10")])), DOC, 50)
        for _ in range(2):
            r = ctx.split_search([sp.split_id], [pl])[0]
            assert not r.kernel_mask & ffi.KERNEL_PREDICATE_FILL
            assert key(r) == key(ref.split_search([sp.split_id], [pl])[0])
        assert ctx.predicate_cache_info()["fills"] == f0
        ctx.set_predicate_cache_budget(0)
        info = ctx.predicate_cache_info()
        assert info["entries"] == 0 and info["used_bytes"] == 0 and info["budget_bytes"] == 0, info
        r = ctx.split_search([sp.split_id], [pl])[0]
        assert not r.kernel_mask & ffi.KERNEL_PREDICATE_FILL and ctx.predicate_cache_info()["entries"] == 0
        ref.close()
    finally:
        ctx.close()


def test_invalidation(corpus):
    ctx = SearcherContext(0)
    try:
        ctx.set_predicate_cache_budget(BUDGET)
        a, b = corpus["col-2049"], CC.small_split(2049, seed=99)
        q = C(CR.bool_([CR.term("d30", SHOULD), CR.term("all", SHOULD), CR.rng("w10", 0, int(np.median(a.cols["w10"].vals)))]))
        pl_a = plan_of(a, q, DOC, 100)
        ctx.register_split(a.img)
        ctx.split_search([a.split_id], [pl_a])
        assert ctx.predicate_cache_info()["entries"] == 1
        # a different image under the same id: the same plan reads the new split
        ctx.unregister_split(a.split_id)
        assert ctx.predicate_cache_info()["entries"] == 0
        ctx.register_split(b.img, split_id=a.split_id)
        r = ctx.split_search([a.split_id], [pl_a])[0]
        assert r.kernel_mask & ffi.KERNEL_PREDICATE_FILL
        assert_same(r, oracle_search(b.img, strip(pl_a)))
        # a split evicted by the residency budget drops its entries
        c = corpus["col-1024"]
        ctx.set_residency_budget(b.img.header().data_len + c.img.header().data_len - 1)
        ctx.register_split(c.img)
        assert not ctx.is_resident(a.split_id)
        info = ctx.predicate_cache_info()
        assert info["entries"] == 0 and info["used_bytes"] == 0, info
    finally:
        ctx.close()


def test_concurrency(corpus):
    ctx = SearcherContext(0)
    try:
        ctx.set_predicate_cache_budget(BUDGET)
        sp = corpus["bool"]
        ctx.register_split(sp.img)
        pl = plan_of(sp, bl([C(bl([body("m00"), ph("title", ["pa", "pb"], SHOULD)])), body("m06", SHOULD)]), BY_U, 100)
        out = [None] * 8
        def go(i):
            out[i] = key(ctx.split_search([sp.split_id], [pl])[0])
        th = [threading.Thread(target=go, args=(i,)) for i in range(8)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        want = key(ctx.split_search([sp.split_id], [pl])[0])
        assert all(o == want for o in out)
        info = ctx.predicate_cache_info()
        assert info["fills"] >= 1 and info["entries"] == 1, info
    finally:
        ctx.close()


# ---- seam A: paging through a leaf search with search_after ------------------------------------------------------
FRACS = [0.2, 0.1, 0.05, 0.05, 0.02]


def leaf(ctx, imgs, q, **kw):
    sreq = proto.enc_search_request(json.dumps(q), **kw)
    lreq = proto.enc_leaf_search_request(sreq, [proto.enc_split_offsets(im.split_id, im.num_docs) for im in imgs], DM)
    return proto.dec_leaf_search_response(ctx.leaf_search(lreq))


def phrase(text):
    return {"type": "full_text", "field": "msg", "text": text, "params": {"mode": {"type": "phrase"}}}


@pytest.mark.parametrize("shape", ["timestamp desc", "two keys", "time range"])
def test_seam_a_paging(shape):
    imgs = [S.synth_split(30_000 + 777 * i, i, FRACS, split_id=f"pc-leaf-{i}", ts_start_secs=1_700_000_000 + 20_000 * i, msg_vocab=64)
            for i in range(3)]
    off, on = SearcherContext(0), SearcherContext(0)
    try:
        on.set_predicate_cache_budget(BUDGET)
        for im in imgs:
            off.register_split(im)
            on.register_split(im)
        q = {"type": "bool", "must": [{"type": "term", "field": "body", "value": "t1"}],
             "should": [phrase("w1 w2"), phrase("w1 w2 w3 w4 w5 w6 w7 w8 w9 w10")],
             "must_not": [{"type": "term", "field": "body", "value": "t3"}]}
        kw = dict(max_hits=100, sort_fields=[("timestamp", 1)])
        if shape == "two keys":
            kw["sort_fields"] = [("tenant_id", 0), ("timestamp", 1)]
        if shape == "time range":
            kw.update(start_timestamp=1_700_000_000 + 5_000, end_timestamp=1_700_000_000 + 50_000)
        page, sa, pages = 0, None, 0
        seen = 0
        while True:
            args = dict(kw, search_after=sa) if sa else kw
            i0 = on.predicate_cache_info()
            a, b = leaf(off, imgs, q, **args), leaf(on, imgs, q, **args)
            i1 = on.predicate_cache_info()
            assert a["num_hits"] == b["num_hits"] and a["partial_hits"] == b["partial_hits"], (shape, page)
            if sa is None:
                assert i1["fills"] == i0["fills"] and i1["misses"] == i0["misses"], (shape, i0, i1)  # no search_after
            elif page == 1:
                assert i1["fills"] - i0["fills"] == len(imgs), (shape, i0, i1)
            else:
                assert i1["fills"] == i0["fills"] and i1["hits"] - i0["hits"] == len(imgs), (shape, page, i0, i1)
            if not b["partial_hits"]:
                break
            if sa is None:
                total = b["num_hits"]
            seen += len(b["partial_hits"])
            sa = b["partial_hits"][-1]
            page += 1
        assert seen == total and page > 20, (shape, seen, total, page)  # the whole order, page by page
        # ranked by _score: never fills
        f0 = on.predicate_cache_info()["fills"]
        first = leaf(on, imgs, q, max_hits=10, sort_fields=[("_score", 1)])
        nxt = leaf(on, imgs, q, max_hits=10, sort_fields=[("_score", 1)], search_after=first["partial_hits"][-1])
        assert nxt["partial_hits"] == leaf(off, imgs, q, max_hits=10, sort_fields=[("_score", 1)], search_after=first["partial_hits"][-1])["partial_hits"]
        assert on.predicate_cache_info()["fills"] == f0
    finally:
        off.close()
        on.close()


# ---- the fuzz generator's bool trees x sort specs, with CACHE nodes at random clauses ---------------------------
from hypothesis import HealthCheck, given, settings, strategies as st  # noqa: E402
import test_gpu_fuzz as F  # noqa: E402
from test_predicate_cache_host import with_cache  # noqa: E402


@pytest.fixture(scope="module")
def fuzz_split():
    return F._clustered_split("pc-fuzz-0")


@settings(max_examples=40, deadline=None, derandomize=True, suppress_health_check=list(HealthCheck))
@given(kids=F._tree(), msm=st.sampled_from([None, None, 1, 2]), sort=F._SORTS, k=st.sampled_from([0, 7, 100, 1000]),
       with_aggs=st.integers(0, 2), seed=st.integers(0, 1 << 30))
def test_fuzz_against_the_oracle(gpu_ctx, fuzz_split, kids, msm, sort, k, with_aggs, seed):
    """Every fuzz plan with CACHE nodes at random clauses: disabled, miss and hit equal the oracle's result for the
    plan without them."""
    img = fuzz_split
    aggs = [F.terms_agg(img, "code"), F.histogram_agg(img, "timestamp", 3600e9)] if with_aggs == 1 else []
    root = F._build(img, kids, msm=msm)
    plain = P.make_plan(root, k, F._sort(img, sort), aggs=aggs)
    cached = P.make_plan(with_cache(root, seed), k, F._sort(img, sort), aggs=aggs)
    want = oracle_search(img, plain)
    ctx = _fuzz_ctx(img)
    ctx.set_predicate_cache_budget(0)
    tag_ = f"kids={kids} msm={msm} sort={sort} k={k} seed={seed}"
    assert_same(ctx.split_search([img.split_id], [cached])[0], want, ctx=tag_ + " disabled")
    ctx.set_predicate_cache_budget(BUDGET)
    for run in ("miss", "hit"):
        assert_same(ctx.split_search([img.split_id], [cached])[0], want, ctx=f"{tag_} {run}")


_FUZZ = {}


def _fuzz_ctx(img):
    if img.split_id not in _FUZZ:
        _FUZZ[img.split_id] = SearcherContext(0)
        _FUZZ[img.split_id].register_split(img)
    return _FUZZ[img.split_id]


def teardown_module():
    for c in _FUZZ.values():
        c.close()
