"""Column sets (QW_NODE_COL_SET) and large text sets on the GPU, bit for bit against a brute force (term_sets_ref's
restatement over column_corpora's source arrays), against the oracle on the plan with every set rewritten as a bool of
its children, and, where the set fits the window program as a bool of RANGE clauses, against that plan on the GPU.

Routes, asserted from `kernel_mask` on every call:
  * k_window scan: a set as the only required clause, over every FULL width 0..64 and the OPTIONAL / MULTI copies, at
    set sizes 1, 2, 31, 32, 33, 1 000 and 65 536 of stored values, values one off them, between gcd multiples and
    outside [min, max]; sets as should (minimum_should_match) and must_not;
  * k_window gather: term AND term AND set;
  * k_driver: term AND 1..4 sets, with doc-id, column and _score sorts at K 0, 10 and 4096, and search_after through a
    whole order;
  * aggregations under a set filter, the predicate cache over a set, malformed COL_SET plans;
  * text: wildcards and term sets of more than 64 terms (KERNEL_TERM_SET), one call over splits of which one converts
    and one does not, and a seam-A leaf request with an ES-style `terms` list of 10 000 ids."""
import json

import numpy as np
import pytest

from quickwit_b200 import ffi, plan as P, splitgen as S
from quickwit_b200.proto import ASC, DESC
from helpers import assert_same
from test_gpu_leaf_search import gpu_root_search
import column_corpora as CC
import column_ref as R
import term_sets_ref as T

pytestmark = pytest.mark.gpu

DRIVER, WINDOW, TERM_SET = ffi.KERNEL_DRIVER, ffi.KERNEL_WINDOW, ffi.KERNEL_TERM_SET
SIZES = (1, 2, 31, 32, 33, 1000)
BOOL_FITS = 66   # queries with up to this many set values also run with each set as a bool of RANGE should clauses


@pytest.fixture(scope="module")
def main(gpu_ctx):
    sp = CC.main_split("ts-cf-main")
    gpu_ctx.register_split(sp.img)
    yield sp
    gpu_ctx.unregister_split(sp.split_id)


def _route_ok(r, route, tag):
    if route == DRIVER:
        assert r.kernel_mask & DRIVER and not r.kernel_mask & WINDOW, tag
    else:
        assert r.kernel_mask & WINDOW and not r.kernel_mask & DRIVER, tag
        assert r.window_docs > 0 or r.num_hits == 0, tag


def _as_bool(q):
    if q.kind == "set":
        return T.SetQ(q.col, q.values, q.occur, as_bool=True)
    if q.kind == "bool":
        return R.bool_([_as_bool(c) for c in q.children], q.msm, q.occur)
    return q


def _set_values(q):
    if q.kind == "set":
        return len(set(q.values))
    return sum(_set_values(c) for c in q.children) if q.kind == "bool" else 0


def _small_sets(q):
    return _set_values(q) <= BOOL_FITS


def run(ctx, items, route, label="", batch=8):
    """items: (Q, Sort, K, search_after, aggs) over the main split; one split_search call per `batch` items."""
    sp = items[0][0]
    out = []
    for i0 in range(0, len(items), batch):
        chunk = items[i0:i0 + batch]
        plans = [T.plan(sp, q, sort, K, sa, aggs) for sp, q, sort, K, sa, aggs in chunk]
        res = ctx.split_search([it[0].split_id for it in chunk], plans)
        twins = [(k, T.plan(sp, _as_bool(q), sort, K, sa, aggs)) for k, (sp, q, sort, K, sa, aggs) in enumerate(chunk)
                 if _small_sets(q)]
        twin_res = dict(zip([k for k, _ in twins], ctx.split_search([chunk[k][0].split_id for k, _ in twins],
                                                                    [p for _, p in twins]))) if twins else {}
        for k, ((sp, q, sort, K, sa, aggs), r, pl) in enumerate(zip(chunk, res, plans)):
            tag = f"{label} {q!r} sort={sort.keys} K={K} kernel_mask={r.kernel_mask:#x}"
            _route_ok(r, route, tag)
            assert_same(r, T.oracle_search(sp.img, pl), ctx=tag)
            R.check(r, sp, q, sort, K, sa, ctx=tag, ev=T.evaluate)
            if k in twin_res:
                w = twin_res[k]
                assert (w.num_hits, [tuple(h[:4]) for h in w.hits]) == (r.num_hits, [tuple(h[:4]) for h in r.hits]), tag + " (bool twin)"
            out.append(r)
    return out


def item(sp, q, sort, K, sa=None, aggs=()):
    return (sp, q, sort, K, sa, aggs)


def _set(sp, name, k, seed, occur=R.FILTER):
    rs = np.random.default_rng(seed)
    return T.SetQ(name, T.probe_values(sp.cols[name], k, rs), occur)


COLUMNS = [f"w{b}" for b in range(65)] + [f"{p}{b}" for b in CC.MC_WIDTHS for p in "om"] + ["g1000", "g3", "i64", "u64", "f64", "dt", "bool"]


def test_scan_every_column_and_size(gpu_ctx, main):
    items = []
    for ci, name in enumerate(COLUMNS):
        for k in SIZES:
            items.append(item(main, R.bool_([_set(main, name, k, 1000 * ci + k)]), R.SORT_DOC_DESC, 10))
    run(gpu_ctx, items, WINDOW, "scan")


def test_scan_65536_values(gpu_ctx, main):
    items = [item(main, R.bool_([_set(main, name, ffi.MAX_SET_TERMS, 7 + i)]), sort, K)
             for i, name in enumerate(("w17", "m10", "g1000"))
             for sort, K in ((R.SORT_DOC_ASC, 4096), (R.col_sort(name, DESC), 10))]
    run(gpu_ctx, items, WINDOW, "scan-65536", batch=4)


def test_should_must_not_and_nested(gpu_ctx, main):
    items = []
    for ci, name in enumerate(("w9", "o31", "m53", "f64", "w40")):
        a, b, c = (_set(main, name, k, 50 * ci + k, R.SHOULD) for k in (33, 1000, 2))
        n = _set(main, "w12", 1000, ci, R.MUST_NOT)
        items += [item(main, R.bool_([a, b, c], msm=2), R.SORT_DOC_DESC, 100),
                  item(main, R.bool_([R.exists(name), n]), R.col_sort(name, ASC), 100),
                  item(main, R.bool_([R.bool_([a, b], occur=R.MUST), R.bool_([n], occur=R.FILTER)]), R.SORT_DOC_ASC, 10)]
    run(gpu_ctx, items, WINDOW, "should/must_not")


def test_gather_after_terms(gpu_ctx, main):
    items = [item(main, R.bool_([R.term(t), R.term("all"), _set(main, name, k, k)]), R.SORT_DOC_DESC, 100)
             for t in R.GATHER_TERMS for name in ("w33", "m64", "o9") for k in (32, 1000)]
    run(gpu_ctx, items, WINDOW, "gather")


def test_driver_filters(gpu_ctx, main):
    items = []
    names = ("w5", "o32", "m11", "i64", "w64")
    for n_f in range(1, 5):
        for k in (2, 33, 1000):
            q = R.bool_([R.term("d30")] + [_set(main, names[(j + n_f) % 5], k, 31 * j + k) for j in range(n_f)])
            for sort, K in ((R.SORT_DOC_DESC, 10), (R.col_sort("w20", ASC), 4096), (R.col_sort("w33", DESC), 10),
                            (R.SORT_DOC_ASC, 0)):
                items.append(item(main, q, sort, K))
    run(gpu_ctx, items, DRIVER, "driver")


def test_score_sort_with_the_set_in_a_filter(gpu_ctx, main):
    sort = R.Sort([(ffi.SORT_SCORE, DESC, None)])
    for K in (0, 10, 4096):
        q = R.bool_([R.term("d30"), _set(main, "w10", 1000, K)])
        sp = main
        pl = T.plan(sp, q, sort, K)
        (r,) = gpu_ctx.split_search([sp.split_id], [pl])
        assert r.kernel_mask & DRIVER, hex(r.kernel_mask)
        assert_same(r, T.oracle_search(sp.img, pl), ctx=f"score K={K}")


def test_paging_through_a_whole_order(gpu_ctx, main):
    for q, route in ((R.bool_([R.term("d30"), _set(main, "w9", 1000, 3)]), DRIVER),
                     (R.bool_([_set(main, "m33", 1000, 4)]), WINDOW)):
        for sort in (R.col_sort("w10", ASC), R.col_sort("o10", DESC)):
            got, sa = [], None
            while True:
                (r,) = run(gpu_ctx, [item(main, q, sort, 4096, sa)], route, "page")
                got += r.hits
                if len(r.hits) < 4096:
                    break
                sa = R.after(r.hits[-1])
            mask, score = T.evaluate(main, q)
            _n, want = R.top_k(main, mask, score, sort, main.num_docs)
            assert [tuple(int(x) for x in h[:4]) for h in got] == want


def test_aggregations_under_a_set_filter(gpu_ctx, main):
    aggs = [R.P.Agg(ffi.AGG_STATS, column=main.ords["w20"])]
    items = [item(main, R.bool_([_set(main, name, k, k)]), R.SORT_DOC_DESC, 10, aggs=aggs)
             for name in ("w15", "m31") for k in (33, 1000)]
    run(gpu_ctx, items, WINDOW, "aggs")


def test_predicate_cache(gpu_ctx, main):
    gpu_ctx.set_predicate_cache_budget(64 << 20)
    try:
        s = _set(main, "w22", 1000, 9)
        root = P.bool_([P.term(main.img, "t", "all"), P.cache(T.node(main, s))])
        pl = P.make_plan(root, 100, R.SORT_DOC_DESC.spec(main), aggs=[R.P.Agg(ffi.AGG_STATS, column=main.ords["w20"])])
        want = T.oracle_search(main.img, pl)
        for _ in range(2):   # a miss fills the entry, a hit reads it
            (r,) = gpu_ctx.split_search([main.split_id], [pl])
            assert_same(r, want, ctx="cache")
        assert gpu_ctx.predicate_cache_info()["hits"] >= 1
    finally:
        gpu_ctx.set_predicate_cache_budget(0)


def test_malformed_col_set_plans(gpu_ctx, main):
    c, c2 = main.ords["w10"], main.ords["w11"]

    def with_kids(kids, occur=ffi.OCCUR_FILTER):
        return P.Node(ffi.NODE_COL_SET, occur, children=kids, column=c)

    def rng(v, col=c, hi=None):
        return P.Node(ffi.NODE_RANGE, ffi.OCCUR_SHOULD, column=col, lo=v, hi=v if hi is None else hi)

    bad = [with_kids([P.Node(ffi.NODE_TERM, ffi.OCCUR_SHOULD, term_ord=0)]), with_kids([rng(5), rng(6, col=c2)]),
           with_kids([rng(5, hi=6)]), with_kids([rng(6), rng(5)]), with_kids([rng(5), rng(5)])]
    plans = [P.make_plan(P.bool_([P.term(main.img, "t", "all"), n]), 10) for n in bad]
    empty = P.make_plan(P.bool_([P.term(main.img, "t", "all")]), 10)
    hs = ffi.QwPlanHeader.from_buffer_copy(empty)
    # E = 0: a COL_SET node without children, written by hand
    nodes = P._flatten(P.bool_([P.term(main.img, "t", "all"), P.Node(ffi.NODE_RANGE, ffi.OCCUR_FILTER, column=c, lo=1, hi=1)]))
    nodes[2].kind = ffi.NODE_COL_SET
    hs.num_nodes = len(nodes)
    plans.append(bytes(hs) + b"".join(bytes(n) for n in nodes))
    scored = P.make_plan(P.bool_([P.term(main.img, "t", "all"), with_kids([rng(5)], ffi.OCCUR_MUST)]), 10,
                         [(ffi.SORT_SCORE, DESC, ffi.ABSENT)])
    for pl, code in [(p, ffi.EINVALID_ARG) for p in plans] + [(scored, ffi.EUNSUPPORTED)]:
        with pytest.raises(ffi.QwGpuError) as e:
            gpu_ctx.split_search([main.split_id], [pl])
        assert e.value.code == code, e.value.msg


# ---- text sets and the compiler's selection, end to end ---------------------------------------------------------------
@pytest.fixture(scope="module")
def text(gpu_ctx):
    docs = T.corpus_docs()
    imgs = [S.build_split(docs, T.MAPPING, "ts-text-a"), S.build_split(docs[:40], T.MAPPING, "ts-text-b")]
    for im in imgs:
        gpu_ctx.register_split(im)
    yield docs, imgs
    for im in imgs:
        gpu_ctx.unregister_split(im.split_id)


def _both(gpu_ctx, imgs, ast, **kw):
    plans = [T.compile_plan(im, ast, T.MAPPING, **kw) for im in imgs]
    res = gpu_ctx.split_search([im.split_id for im in imgs], plans)
    for im, pl, r in zip(imgs, plans, res):
        assert_same(r, T.oracle_search(im, pl), ctx=f"{ast} {im.split_id}")
    return plans, res


def test_text_sets_over_64_terms(gpu_ctx, text):
    docs, imgs = text
    for ast, want in ((T.wildcard("raw", "r1*"), [d["raw"].startswith("r1") for d in docs]),
                      (T.term_set({"raw": [f"r{k:03d}" for k in range(0, 400, 3)]}), [int(d["raw"][1:]) % 3 == 0 for d in docs]),
                      (T.term_set({"ipi": [f"10.0.0.{k}" for k in range(200)]}), [d["ipi"].startswith("10.0.0.") and int(d["ipi"].split(".")[3]) < 200 for d in docs]),
                      (T.term_set({"ipf": [f"192.168.1.{k}" for k in range(256)]}), [d["ipf"].startswith("192.168.1.") for d in docs])):
        plans, (ra,) = _both(gpu_ctx, imgs[:1], ast, max_hits=T.N_DOCS)
        assert T.set_nodes(plans[0]), ast
        if any(n.kind == ffi.NODE_TERM_SET for n in T.set_nodes(plans[0])):
            assert ra.kernel_mask & TERM_SET, hex(ra.kernel_mask)
        assert np.array_equal(T.hit_mask(ra, T.N_DOCS), np.array(want)), ast


def test_one_call_over_a_converted_and_an_unconverted_split(gpu_ctx, text):
    docs, imgs = text
    plans, res = _both(gpu_ctx, imgs, T.wildcard("raw", "r1*"), max_hits=100)
    assert T.set_nodes(plans[0]) and not T.set_nodes(plans[1])
    assert res[0].kernel_mask & TERM_SET


def test_seam_a_terms_list_of_10000_ids(gpu_ctx):
    docs = [{"id": 3 * d + 1, "svc": f"api{d % 5}"} for d in range(40_000)]
    mapping = {"field_mappings": [{"name": "id", "type": "u64", "fast": True}, {"name": "svc", "type": "text", "tokenizer": "raw"}]}
    img = S.build_split(docs, mapping, "ts-ids")
    gpu_ctx.register_split(img)
    try:
        ids = [int(x) for x in np.random.default_rng(5).integers(0, 130_000, size=10_000)]
        ast = {"type": "bool", "must": [{"type": "term", "field": "svc", "value": "api1"}], "filter": [T.term_set({"id": ids})]}
        got, _leaf = gpu_root_search(gpu_ctx, [img], ast, mapping, max_hits=50, sort_fields=[("id", 1)])
        want = T.cpu_root_search([img], ast, mapping, max_hits=50, sort_fields=[("id", 1)])
        assert got["num_hits"] == want["num_hits"] and got["partial_hits"] == want["partial_hits"]
        idset = set(ids)
        assert got["num_hits"] == sum(d["svc"] == "api1" and d["id"] in idset for d in docs)
    finally:
        gpu_ctx.unregister_split(img.split_id)
