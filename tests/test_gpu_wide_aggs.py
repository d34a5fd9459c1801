"""Aggregation plans of 9 to 32 nodes on the GPU, at most 8 levels deep, reading up to 32 aggregation columns beside 16
query and sort columns. Every call is checked against the brute force (agg_ref for dense cells, hashed_ref /
percentiles_ref for hashed entries, composite_ref for composite pages) and, where the dense layout is small enough,
against the CPU oracle; f64 sums within the summation bound agg_ref checks. Every call also asserts the kernel route
from kernel_mask: the dense generic path, the fast path, the hashed walk with its capacity re-run and the composite
cut all serve wide plans, and a flat match-all plan of more than 8 nodes leaves k_aggscan for k_window."""
import json

import numpy as np
import pytest

from quickwit_b200 import ffi, plan as P, proto, service
from oracle import oracle as O
from agg_ref import assert_cells, cells
from agg_ref import _layout
from hashed_ref import assert_entries, sparse_cells
import composite_ref as CR
import percentiles_ref as PR
import pipeline as PL
import wide_aggs_cases as W

pytestmark = pytest.mark.gpu

AGGSCAN, WINDOW, FAST = ffi.KERNEL_AGGSCAN, ffi.KERNEL_WINDOW, ffi.KERNEL_FAST_AGGS
HASHED, RETRY, CUT = ffi.KERNEL_HASHED_AGGS, ffi.KERNEL_HASHED_AGGS_RETRY, ffi.KERNEL_COMPOSITE_CUT


@pytest.fixture(scope="module")
def corpus(gpu_ctx):
    rng = np.random.default_rng(17)
    c = {"main": W.WideSplit("wide-main", W.make_docs(12_001, 1)),
         "many": [W.WideSplit(f"wide-many-{i}", W.make_docs(int(n), 200 + i)) for i, n in enumerate(rng.integers(1, 3000, 40))]}
    for sp in [c["main"]] + c["many"]:
        gpu_ctx.register_split(sp.img)
    yield c
    for sp in [c["main"]] + c["many"]:
        gpu_ctx.unregister_split(sp.img.split_id)


def _query(sp, mode):
    """(root, max_hits, sort, matched docs or None) of a query mode: count-only match_all, K = 10 by the `t` column,
    K = 10 by _score under a term query."""
    if mode == "count":
        return P.bool_([P.match_all()]), 0, ((ffi.SORT_DOCID, ffi.ORDER_DESC, ffi.ABSENT),), None
    if mode == "by_t":
        return P.bool_([P.match_all()]), 10, ((ffi.SORT_COLUMN, ffi.ORDER_DESC, sp.by_name["t"]),), None
    docs = [i for i, d in enumerate(sp.docs) if "b" in d["body"].split()]
    return P.bool_([P.term(sp.img, "body", "b")]), 10, ((ffi.SORT_SCORE, ffi.ORDER_DESC, ffi.ABSENT),), docs


def _run(ctx, jobs, mode="count"):
    """jobs: [(split, aggs)] in one call; every result checked against the brute force and the oracle (dense layout
    where it is small enough), hits against the oracle's."""
    qs = [_query(sp, mode) for sp, _a in jobs]
    plans = [P.make_plan(root, k, sort, aggs=aggs) for (sp, aggs), (root, k, sort, _d) in zip(jobs, qs)]
    got = ctx.split_search([sp.img.split_id for sp, _a in jobs], plans)
    for (sp, aggs), plan, (_r, _k, _s, docs), r in zip(jobs, plans, qs, got):
        tag = f"{sp.img.split_id} ({W.count_nodes(aggs)} nodes, {mode}) kernel_mask={r.kernel_mask:#x}"
        hashed, _bound = service.agg_layout(sp.img, plan)
        ref = O.split_search(sp.img, plan)
        assert r.num_hits == ref.num_hits and r.hits == ref.hits, tag
        if hashed:
            assert r.cells == [] and r.kernel_mask & HASHED, tag
            assert_entries(r.entries, sparse_cells(aggs, sp.cols, docs), tag)
        else:
            assert r.entries == [], tag
            want = cells(aggs, sp.cols, docs)
            assert_cells(r.cells, want, tag)
            assert_cells(ref.cells, want, f"{tag}: oracle")
        assert r.kernel_mask & WINDOW and not r.kernel_mask & AGGSCAN, tag
    return got


# ---- dense generic path ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["count", "by_t", "by_score"])
@pytest.mark.parametrize("levels", [1, 2, 3])
@pytest.mark.parametrize("n", [9, 16, 32])
def test_dense_generic(gpu_ctx, corpus, n, levels, mode):
    sp = corpus["main"]
    aggs = W.dense_tree(sp, n, levels)
    got = _run(gpu_ctx, [(sp, aggs)], mode)
    assert not got[0].kernel_mask & (FAST | HASHED), hex(got[0].kernel_mask)
    assert got[0].cells


# ---- fast path -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["count", "by_t"])
@pytest.mark.parametrize("n", [9, 17, 32])
def test_fast_path(gpu_ctx, corpus, n, mode):
    sp = corpus["main"]
    aggs = W.fast_plan(sp, n)
    assert sum(x for *_a, x in _layout(aggs)) <= 4096
    got = _run(gpu_ctx, [(sp, aggs)], mode)
    assert got[0].kernel_mask & FAST, hex(got[0].kernel_mask)


# ---- a match-all flat plan over 8 nodes leaves k_aggscan -------------------------------------------------------------
def test_flat_match_all_leaves_aggscan(gpu_ctx, corpus):
    sp = corpus["main"]
    nine = W.aggscan_flat(sp, 9)
    wide = _run(gpu_ctx, [(sp, nine)])[0]
    assert wide.kernel_mask & WINDOW and not wide.kernel_mask & AGGSCAN, hex(wide.kernel_mask)
    # the first 8 nodes alone stay on k_aggscan and agree with the wide call node for node
    eight = W.aggscan_flat(sp, 8)
    plan = P.make_plan(P.bool_([P.match_all()]), 0, aggs=eight)
    narrow = gpu_ctx.split_search([sp.img.split_id], [plan])[0]
    assert narrow.kernel_mask & AGGSCAN and not narrow.kernel_mask & WINDOW, hex(narrow.kernel_mask)
    assert_cells(narrow.cells, cells(eight, sp.cols), "8 nodes on k_aggscan")
    assert narrow.cells == wide.cells[:len(narrow.cells)]


# ---- hashed walk -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [9, 16, 32])
def test_hashed_eight_levels(gpu_ctx, corpus, n):
    sp = corpus["main"]
    aggs = W.hashed_tree(sp, n)
    got = _run(gpu_ctx, [(sp, aggs)])
    assert not got[0].kernel_mask & RETRY and got[0].entries


def test_hashed_with_hits(gpu_ctx, corpus):
    sp = corpus["main"]
    _run(gpu_ctx, [(sp, W.hashed_tree(sp, 32))], "by_score")


def test_hashed_percentiles(gpu_ctx):
    """An 8-level chain of bucket nodes above a percentiles leaf, with percentiles siblings, 32 nodes (over 3000 docs:
    the chain's bound on distinct cells grows with the docs and the bins)."""
    sp = W.WideSplit("wide-pct", W.make_docs(3000, 9))
    gpu_ctx.register_split(sp.img)

    def pct(name, missing=None):
        return P.percentiles(sp.by_name[name], PR.num_bins(sp.col(name)), missing)

    tops = [W.chain(sp, 7, pct("lat"), ranges=False)]
    while W.count_nodes(tops) < 32:
        i = len(tops)
        tops.append(pct(("latf", "optf", "lat")[i % 3], missing=1.5 if i % 3 == 1 else None) if i % 2 else
                    sp.terms("svc", children=[pct("latf")]))
    tops = tops[:-1] if W.count_nodes(tops) > 32 else tops
    assert W.count_nodes(tops) == 32 and W.depth_of(tops) == 8
    plan = P.make_plan(P.bool_([P.match_all()]), 0, aggs=tops)
    try:
        r = gpu_ctx.split_search([sp.img.split_id], [plan])[0]
    finally:
        gpu_ctx.unregister_split(sp.img.split_id)
    assert r.kernel_mask & HASHED and r.kernel_mask & WINDOW and not r.kernel_mask & AGGSCAN, hex(r.kernel_mask)
    assert_entries(r.entries, PR.entries(plan, sp.cols), "percentiles")


def test_hashed_capacity_rerun(gpu_ctx):
    """Wide trees whose distinct cells outgrow the initial table capacity run again at the bound."""
    sp = W.WideSplit("wide-rerun", W.make_docs(40_000, 5))
    gpu_ctx.register_split(sp.img)
    try:
        # the 8-level chain over 40 000 docs and terms over the near-unique `t` column: more than 65536 cells in all
        aggs = W.hashed_tree(sp, 29, leaf="lat") + [sp.terms("t", children=[sp.terms("k00", children=[sp.stats("lat")])])]
        got = _run(gpu_ctx, [(sp, aggs)])
        assert got[0].kernel_mask & RETRY and len(got[0].entries) > ffi.HASHED_INIT_CELLS, hex(got[0].kernel_mask)
    finally:
        gpu_ctx.unregister_split(sp.img.split_id)


# ---- composites: 9, 16 and 32 source nodes, paged to the end ------------------------------------------------------------
def _composites(n_sources):
    """Composites of at most 8 sources each (a composite's sources are levels of its chain) adding up to n_sources."""
    fields = ["svc", "k00", "k01", "opt", "k02", "tags", "k03", "k04", "k05", "k06", "lvl", "k07"]
    out, used = {}, 0
    while used < n_sources:
        m = min(8, n_sources - used)
        srcs = []
        for j in range(m):
            f = fields[(used + j) % len(fields)]
            body = {"terms": {"field": f, "order": "desc" if (used + j) % 3 == 1 else "asc"}}
            if f in ("opt", "tags", "lvl"):
                body["terms"]["missing_bucket"] = True
            srcs.append({f"s{used + j}": body})
        out[f"c{len(out)}"] = {"size": 400, "sources": srcs}
        used += m
    return out


@pytest.mark.parametrize("n_sources", [9, 16, 32])
def test_composites_paged(gpu_ctx, corpus, n_sources):
    splits = corpus["many"][:4]
    specs = _composites(n_sources)
    docs = [d for sp in splits for d in sp.docs]
    want = {name: CR.as_json(CR.all_buckets(docs, spec), spec) for name, spec in specs.items()}
    got = {name: [] for name in specs}
    after = {}
    dm = json.dumps(W.MAPPING)
    for _ in range(max(len(v) for v in want.values()) // 400 + 2):
        live = {nm: (dict(s, after=after[nm]) if nm in after else s) for nm, s in specs.items() if after.get(nm, 0) is not None}
        if not live:
            break
        req = PL.search_request(PL.MATCH_ALL, max_hits=0, aggs={nm: {"composite": s} for nm, s in live.items()})
        plans = [service.compile_plan(sp.img, req, dm) for sp in splits]
        res = gpu_ctx.split_search([sp.img.split_id for sp in splits], plans)
        for r in res:
            assert r.kernel_mask & HASHED and r.kernel_mask & CUT and not r.kernel_mask & AGGSCAN, hex(r.kernel_mask)
        parts = [service.build_leaf_response_entries(sp.img, req, dm, r.num_hits, r.hits, r.entries) for sp, r in zip(splits, res)]
        merged = proto.dec_leaf_search_response(service.merge_leaf_responses(req, parts))
        page = json.loads(service.finalize_aggregation(json.dumps({nm: {"composite": s} for nm, s in live.items()}),
                                                       merged["intermediate_aggregation_result"] or b""))
        for nm in live:
            got[nm] += page[nm]["buckets"]
            after[nm] = page[nm]["after_key"] if page[nm]["buckets"] else None
    assert all(v is None for v in after.values())
    assert got == want


# ---- columns: 32 aggregation columns beside 16 query and sort columns ---------------------------------------------------
def _wide_columns(sp, n_query, n_agg):
    """A plan whose query filters on n_query - 1 columns and sorts by one more, and whose 32 aggregation nodes read
    n_agg other columns (stats nodes over k16.., then histograms over the same columns)."""
    ks = [f"k{i:02d}" for i in range(W.K_COLS)]
    root = P.bool_([P.range_(sp.img, c, 0, 1 << 40, occur=ffi.OCCUR_FILTER) for c in ks[:n_query - 1]])
    sort = ((ffi.SORT_COLUMN, ffi.ORDER_ASC, sp.by_name["lat"]),)
    a_cols = (ks[16:] + ["code", "latf", "t"])[:n_agg]
    aggs = [sp.stats(c) for c in a_cols] + [sp.hist(c, 1.0) for c in a_cols[:max(0, 32 - n_agg)]]
    return root, sort, aggs


def test_column_budget(gpu_ctx, corpus):
    sp = corpus["main"]
    root, sort, aggs = _wide_columns(sp, 16, 32)
    plan = P.make_plan(root, 10, sort, aggs=aggs)
    r = gpu_ctx.split_search([sp.img.split_id], [plan])[0]
    ref = O.split_search(sp.img, plan)
    assert r.hits == ref.hits and r.num_hits == ref.num_hits == sp.num_docs
    assert_cells(r.cells, cells(aggs, sp.cols), "16 query and sort columns, 32 aggregation columns")
    # one more aggregation column, then one more query column: refused, and the context serves the next request
    for (root2, sort2, aggs2), msg in ((_over_aggs(sp), "more than 32 aggregation nodes"),
                                       (_wide_columns(sp, 17, 32), "plan uses more than 16 columns")):
        with pytest.raises(ffi.QwGpuError) as e:
            gpu_ctx.split_search([sp.img.split_id], [P.make_plan(root2, 10, sort2, aggs=aggs2)])
        assert e.value.code == ffi.EUNSUPPORTED and msg in e.value.msg, e.value.msg
        again = gpu_ctx.split_search([sp.img.split_id], [plan])[0]
        assert again.hits == r.hits and again.cells == r.cells


def _over_aggs(sp):
    """33 aggregation columns beside the 16 of the query and sort: every node reads one column, so they take 33 nodes."""
    root, sort, _a = _wide_columns(sp, 16, 32)
    cols = [f"k{i:02d}" for i in range(16, W.K_COLS)] + ["code", "latf", "t"]
    return root, sort, [sp.stats(c) for c in cols[:33]]


# ---- limits ----------------------------------------------------------------------------------------------------------
def test_node_and_level_limits(gpu_ctx, corpus):
    sp = corpus["main"]
    root = P.bool_([P.match_all()])
    for aggs, ok in ((W.dense_tree(sp, 32, 2), True), (W.dense_tree(sp, 33, 2), False),
                     (W.hashed_tree(sp, 8, 8), True), ([W.chain(sp, 8, sp.stats("lat"))], False)):
        plan = P.make_plan(root, 0, aggs=aggs)
        if ok:
            _run(gpu_ctx, [(sp, aggs)])
            continue
        with pytest.raises(ffi.QwGpuError) as e:
            gpu_ctx.split_search([sp.img.split_id], [plan])
        assert e.value.code == ffi.EUNSUPPORTED, e.value.msg
        assert ("more than 32 aggregation nodes" if W.count_nodes(aggs) > 32 else "more than 8 levels") in e.value.msg


# ---- mixed batch -----------------------------------------------------------------------------------------------------
def test_mixed_batch(gpu_ctx, corpus):
    """40 splits in one call, every other one with a 32-node plan; the 8-node plans' cells equal those of a call without
    the wide plans (bit for bit but for the order of f64 sums)."""
    many = corpus["many"]
    jobs = [(sp, W.dense_tree(sp, 32, 2) if i % 2 else W.dense_tree(sp, 8, 2)) for i, sp in enumerate(many)]
    mixed = _run(gpu_ctx, jobs)
    narrow_jobs = [j for i, j in enumerate(jobs) if i % 2 == 0]
    alone = gpu_ctx.split_search([sp.img.split_id for sp, _a in narrow_jobs],
                                 [P.make_plan(P.bool_([P.match_all()]), 0, aggs=a) for _s, a in narrow_jobs])
    for (sp, aggs), a, b in zip(narrow_jobs, alone, mixed[0::2]):
        assert_cells(a.cells, cells(aggs, sp.cols), sp.img.split_id)
        for x, y, w in zip(a.cells, b.cells, cells(aggs, sp.cols), strict=True):
            # (an f64 sum takes its atomics in the order of the call's warps: only exact sums compare bit for bit)
            assert x == y if w.sum is None or w.sum.exact else (x[0], x[2], x[3]) == (y[0], y[2], y[3])


# ---- end to end: the 10-node dashboard request ------------------------------------------------------------------------
def _by_service(metrics):
    return {"terms": {"field": "svc"}, "aggs": {"per_minute": {"date_histogram": {"field": "ts", "fixed_interval": "1m"},
                                                               "aggs": metrics}}}


LAT = {"lat_avg": {"avg": {"field": "lat"}}, "lat_min": {"min": {"field": "lat"}}, "lat_max": {"max": {"field": "lat"}},
       "lat_pct": {"percentiles": {"field": "lat"}}}
BYTES = {"bytes_sum": {"sum": {"field": "code"}}, "bytes_avg": {"avg": {"field": "code"}}}
OTHERS = {"over_time": {"date_histogram": {"field": "ts", "fixed_interval": "10m"}}, "by_status": {"terms": {"field": "opt"}}}
DASHBOARD = {"by_service": _by_service({**LAT, **BYTES}), **OTHERS}  # 10 nodes


def _leaf_json(ctx, splits, aggs):
    dm = json.dumps(W.MAPPING)
    req = PL.search_request(PL.MATCH_ALL, max_hits=0, aggs=aggs)
    lreq = proto.enc_leaf_search_request(req, [proto.enc_split_offsets(sp.img.split_id, sp.num_docs) for sp in splits], dm)
    leaf = proto.dec_leaf_search_response(ctx.leaf_search(lreq))
    assert not leaf.get("failed_splits"), leaf.get("failed_splits")
    return json.loads(service.finalize_aggregation(json.dumps(aggs), leaf["intermediate_aggregation_result"]))


def test_dashboard_end_to_end(gpu_ctx, corpus):
    splits = corpus["many"][5:11]
    got = _leaf_json(gpu_ctx, splits, DASHBOARD)
    # every node but the percentiles against the CPU pipeline (oracle cells), the percentiles against their brute force
    no_pct = {"by_service": _by_service({**{k: v for k, v in LAT.items() if k != "lat_pct"}, **BYTES}), **OTHERS}
    want = PL.cpu_root_search([sp.img for sp in splits], PL.MATCH_ALL, W.MAPPING, max_hits=0, aggs=no_pct)["aggregations"]
    docs = [d for sp in splits for d in sp.docs]
    stripped = json.loads(json.dumps(got))
    for b in stripped["by_service"]["buckets"]:
        for m in b["per_minute"]["buckets"]:
            pct = m.pop("lat_pct")
            if m["doc_count"]:
                vals = [float(d["lat"]) for d in docs if d["svc"] == b["key"] and d["ts"] // 60 * 60000 == int(m["key"])]
                assert len(vals) == m["doc_count"] and pct == {"values": PR.expected_values(PR.sketch_of(vals))}
    assert stripped == want
    # the same nodes as two requests of at most 8 nodes each, their JSON joined bucket by bucket
    first = _leaf_json(gpu_ctx, splits, {"by_service": _by_service(LAT), **OTHERS})  # 8 nodes
    second = _leaf_json(gpu_ctx, splits, {"by_service": _by_service(BYTES)})          # 4 nodes
    for b0, b1 in zip(first["by_service"]["buckets"], second["by_service"]["buckets"], strict=True):
        assert b0["key"] == b1["key"]
        for m0, m1 in zip(b0["per_minute"]["buckets"], b1["per_minute"]["buckets"], strict=True):
            m0.update(m1)
    assert first == got
