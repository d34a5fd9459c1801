"""Composite aggregations on the GPU: the hashed walk with the `after` filter (k_window's hashed collect), then the
host's entries builder, merge and finalisation, against composite_ref's brute force from the documents. Every call's
kernel_mask must show the hashed walk and k_composite_cut, and never k_aggscan; every split must return exactly its
first `size` tuples after `after` as leaves, with the chain entries above them."""
import json

import numpy as np
import pytest

from quickwit_b200 import ffi, proto, service, splitgen as S
from quickwit_b200.service import SearcherContext
import composite_ref as R
import pipeline as PL
from test_oracle_goldens import AGG_MAPPING, AGG_SPLIT1, AGG_SPLIT2

pytestmark = pytest.mark.gpu

HASHED, RETRY, AGGSCAN, CUT = ffi.KERNEL_HASHED_AGGS, ffi.KERNEL_HASHED_AGGS_RETRY, ffi.KERNEL_AGGSCAN, ffi.KERNEL_COMPOSITE_CUT
T0 = 1_700_000_000
MAPPING = {"field_mappings": [{"name": "svc", "type": "text", "tokenizer": "raw", "fast": True},
                              {"name": "tags", "type": "u64", "fast": True},
                              {"name": "lat", "type": "u64", "fast": True},
                              {"name": "uid", "type": "u64", "fast": True},
                              {"name": "ts", "type": "datetime", "fast": True, "fast_precision": "seconds"}],
           "timestamp_field": "ts"}


def _docs(n, seed, uid=False):
    rng = np.random.default_rng(seed)
    svc = rng.integers(0, 9, size=n)
    lat = rng.integers(0, 5000, size=n)
    ts = T0 + rng.integers(0, 12 * 3600, size=n)
    k = rng.integers(0, 3, size=n)
    docs = []
    for i in range(n):
        d = {"lat": int(lat[i]), "ts": int(ts[i])}
        if svc[i] < 8:
            d["svc"] = f"service-{int(svc[i])}"
        if k[i]:
            d["tags"] = sorted({int(x) for x in rng.integers(0, 6, size=int(k[i]))})
        if uid:
            d["uid"] = i
        docs.append(d)
    return docs


@pytest.fixture(scope="module")
def ctx():
    c = SearcherContext(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def corpus(ctx):
    splits = []
    for s in range(8):
        docs = _docs(60_000, 100 + s)
        img = S.build_split(docs, MAPPING, f"comp-{s}")
        ctx.register_split(img)
        splits.append((img, docs))
    return splits


@pytest.fixture(scope="module")
def golden(ctx):
    out = []
    for docs, sid in ((AGG_SPLIT1, "comp-golden-1"), (AGG_SPLIT2, "comp-golden-2")):
        img = S.build_split(docs, AGG_MAPPING, sid)
        ctx.register_split(img)
        out.append((img, docs))
    return out


def _search(ctx, splits, aggs, mapping, query=PL.MATCH_ALL, max_hits=0):
    """split_search on the GPU -> per-split leaf responses -> leaf merge -> finalised aggregations; returns
    (aggregations, per-split results)"""
    req = PL.search_request(query, max_hits=max_hits, aggs=aggs)
    dm = json.dumps(mapping)
    plans = [service.compile_plan(img, req, dm) for img, _d in splits]
    res = ctx.split_search([img.split_id for img, _d in splits], plans)
    parts = []
    for (img, _d), r in zip(splits, res):
        assert r.kernel_mask & HASHED and r.kernel_mask & CUT and not r.kernel_mask & AGGSCAN, hex(r.kernel_mask)
        parts.append(service.build_leaf_response_entries(img, req, dm, r.num_hits, r.hits, r.entries))
    merged = proto.dec_leaf_search_response(service.merge_leaf_responses(req, parts))
    return json.loads(service.finalize_aggregation(json.dumps(aggs), merged["intermediate_aggregation_result"] or b"")), res


GOLDEN = {"size": 5, "sources": [{"host": {"terms": {"field": "host", "missing_bucket": True}}},
                                 {"name": {"terms": {"field": "name"}}},
                                 {"response": {"histogram": {"field": "response", "interval": 50}}}]}


def test_rest_goldens(ctx, golden):
    got, _ = _search(ctx, golden, {"c": {"composite": GOLDEN}}, AGG_MAPPING)
    assert got["c"]["buckets"] == [
        {"key": {"host": None, "name": "Bernhard", "response": 100.0}, "doc_count": 1},
        {"key": {"host": None, "name": "Fritz", "response": 0.0}, "doc_count": 2},
        {"key": {"host": "192.168.0.1", "name": "Fred", "response": 100.0}, "doc_count": 1},
        {"key": {"host": "192.168.0.1", "name": "Fritz", "response": 0.0}, "doc_count": 1},
        {"key": {"host": "192.168.0.10", "name": "Albert", "response": 100.0}, "doc_count": 1}]
    assert got["c"]["after_key"] == {"host": "str:192.168.0.10", "name": "str:Albert", "response": "f64:100"}
    nxt, _ = _search(ctx, golden, {"c": {"composite": dict(GOLDEN, after=got["c"]["after_key"])}}, AGG_MAPPING)
    assert nxt["c"]["buckets"] == [
        {"key": {"host": "192.168.0.10", "name": "Holger", "response": 0.0}, "doc_count": 1},
        {"key": {"host": "192.168.0.10", "name": "Werner", "response": 0.0}, "doc_count": 1},
        {"key": {"host": "192.168.0.11", "name": "Manfred", "response": 100.0}, "doc_count": 1}]


def _spec(size, desc):
    o = "desc" if desc else "asc"
    return {"size": size, "sources": [{"svc": {"terms": {"field": "svc", "order": o}}},
                                      {"tags": {"terms": {"field": "tags", "missing_bucket": True, "order": "asc" if desc else "desc"}}},
                                      {"hour": {"date_histogram": {"field": "ts", "fixed_interval": "1h", "order": o}}}]}


_ORDERS = {}


def _check_cut(split_results, splits, spec, after):
    """Each split returned its first `size` tuples after `after` as leaves, and exactly the chain entries above them
    (the composite is the plan's only aggregation: sources are nodes 0..n-1)."""
    srcs = R.sources_of(spec)
    n = len(srcs)
    for (img, ds), r in zip(splits, split_results):
        ck = (img.split_id, json.dumps(spec["sources"]))
        if ck not in _ORDERS:
            _ORDERS[ck] = R.all_buckets(ds, spec)
        mine = _ORDERS[ck]
        if after is not None:
            a = tuple(R.plain_after(after[nm]) for nm, _t, _p in srcs)
            mine = [b for b in mine if R.tuple_cmp(srcs, b[0], a) > 0]
        kept = [k for k, _d in mine[:spec["size"]]]
        per_node = [sum(1 for e in r.entries if e[0] == lvl) for lvl in range(n)]
        assert per_node == [len({k[:lvl + 1] for k in kept}) for lvl in range(n)], (img.split_id, per_node)


def _page_all(ctx, splits, spec, mapping=MAPPING):
    docs = [d for _img, ds in splits for d in ds]
    want = R.as_json(R.all_buckets(docs, spec), spec)
    got, after = [], None
    for _ in range(len(want) // spec["size"] + 2):
        s = spec if after is None else dict(spec, after=after)
        page, res = _search(ctx, splits, {"c": {"composite": s}}, mapping)
        _check_cut(res, splits, spec, after)
        got += page["c"]["buckets"]
        if not page["c"]["buckets"]:
            assert page["c"]["after_key"] == {}
            break
        after = page["c"]["after_key"]
    assert got == want


@pytest.mark.parametrize("size", [7, 1000])
@pytest.mark.parametrize("desc", [False, True])
def test_paging_to_exhaustion(ctx, corpus, size, desc):
    _page_all(ctx, corpus, _spec(size, desc))


@pytest.mark.parametrize("desc", [False, True])
def test_paging_to_exhaustion_size_one(ctx, desc):
    splits = []
    for s in range(3):
        docs = [d for d in _docs(3000, 300 + s) if d["ts"] < T0 + 3 * 3600]
        img = S.build_split(docs, MAPPING, f"comp-small-{int(desc)}-{s}")
        ctx.register_split(img)
        splits.append((img, docs))
    _page_all(ctx, splits, _spec(1, desc))
    for img, _d in splits:
        ctx.unregister_split(img.split_id)


def test_plan_helper_chain(ctx, corpus):
    """A chain built with plan.composite straight into split_search: the cut keeps the `size` first raw tuples
    (svc ascending, null tags last under the descending tags source)."""
    from quickwit_b200 import plan as P
    img, docs = corpus[0]
    svc, tags = img.column_ord("svc"), img.column_ord("tags")
    chain = P.composite([P.Agg(ffi.AGG_TERMS, column=svc, num_buckets=0xFFFFFFFF),
                         P.Agg(ffi.AGG_TERMS, column=tags, num_buckets=0xFFFFFFFF, missing=0)], size=5, desc=[1])
    r = ctx.split_search([img.split_id], [P.make_plan(P.match_all(), 0, aggs=[chain])])[0]
    assert r.kernel_mask & CUT and r.kernel_mask & HASHED
    dict_svc = [b.decode() for b in img.dictionary(svc)]
    sv, ts = img.columns()[svc], img.columns()[tags]
    tuples = {(dict_svc.index(d["svc"]), t) for d in docs if "svc" in d for t in (d.get("tags") or [None])}
    order = sorted(tuples, key=lambda k: (k[0], k[1] is None, -(k[1] or 0)))
    e = r.entries
    leaves = {(e[x[1]][2] * sv.gcd + sv.min_value, None if x[3] else x[2] * ts.gcd + ts.min_value) for x in e if x[0] == 1}
    assert leaves == set(order[:5])


def test_sub_aggregations_and_sibling(ctx, corpus):
    spec = _spec(50, False)
    spec["after"] = {"svc": "str:service-3", "tags": None, "hour": 0}
    aggs = {"c": {"composite": spec, "aggs": {"a": {"avg": {"field": "lat"}}, "s": {"stats": {"field": "lat"}},
                                              "t": {"terms": {"field": "tags"}, "aggs": {"ta": {"avg": {"field": "lat"}}}}}},
            "sib": {"terms": {"field": "svc", "size": 20}}}
    got, _ = _search(ctx, corpus, aggs, MAPPING)
    docs = [d for _i, ds in corpus for d in ds]
    want = R.page(docs, spec)
    assert len(got["c"]["buckets"]) == len(want) == 50
    for b, (k, ds) in zip(got["c"]["buckets"], want):
        assert tuple(b["key"].values()) == k and b["doc_count"] == len(ds)
        lats = [d["lat"] for d in ds]
        assert b["s"]["count"] == len(lats) and b["s"]["min"] == min(lats) and b["s"]["max"] == max(lats)
        assert b["s"]["sum"] == float(sum(lats)) and b["a"]["value"] == pytest.approx(sum(lats) / len(lats), rel=1e-12)
        tags = {}
        for d in ds:
            for t in d.get("tags", []):
                tags.setdefault(t, []).append(d["lat"])
        assert {t["key"]: (t["doc_count"], t["ta"]["value"]) for t in b["t"]["buckets"]} == \
               pytest.approx({t: (len(v), sum(v) / len(v)) for t, v in tags.items()}, rel=1e-12)
    # the sibling equals the same terms aggregation alone (which takes the dense layout)
    alone = PL.search_request(PL.MATCH_ALL, max_hits=0, aggs={"sib": aggs["sib"]})
    dm = json.dumps(MAPPING)
    plans = [service.compile_plan(img, alone, dm) for img, _d in corpus]
    res = ctx.split_search([img.split_id for img, _d in corpus], plans)
    parts = [service.build_leaf_response(img, alone, dm, r.num_hits, r.hits, r.cells) for (img, _d), r in zip(corpus, res)]
    merged = proto.dec_leaf_search_response(service.merge_leaf_responses(alone, parts))
    assert json.loads(service.finalize_aggregation(json.dumps({"sib": aggs["sib"]}), merged["intermediate_aggregation_result"]))["sib"] == got["sib"]


def test_query_with_hits(ctx, corpus):
    img, docs = corpus[0]
    q = PL.bool_(must=[PL.term("svc", "service-2"), {"type": "range", "field": "lat", "lower_bound": {"Included": 1000},
                                                       "upper_bound": {"Excluded": 3000}}])
    spec = _spec(20, True)
    got, res = _search(ctx, [(img, docs)], {"c": {"composite": spec}}, MAPPING, query=q, max_hits=10)
    match = [d for d in docs if d.get("svc") == "service-2" and 1000 <= d["lat"] < 3000]
    assert got["c"]["buckets"] == R.as_json(R.page(match, spec), spec)
    assert res[0].num_hits == len(match)
    plain = ctx.split_search([img.split_id], [service.compile_plan(img, PL.search_request(q, max_hits=10), json.dumps(MAPPING))])[0]
    assert res[0].hits == plain.hits and res[0].num_hits == plain.num_hits


def test_more_tuples_than_the_initial_capacity(ctx):
    docs = _docs(90_000, 7, uid=True)
    img = S.build_split(docs, MAPPING, "comp-wide")
    ctx.register_split(img)
    spec = {"size": 1000, "sources": [{"u": {"terms": {"field": "uid"}}}, {"s": {"terms": {"field": "svc", "missing_bucket": True}}}]}
    got, res = _search(ctx, [(img, docs)], {"c": {"composite": spec}}, MAPPING)
    assert res[0].kernel_mask & RETRY
    assert got["c"]["buckets"] == R.as_json(R.page(docs, spec), spec)
    spec["after"] = got["c"]["after_key"]
    got, res = _search(ctx, [(img, docs)], {"c": {"composite": spec}}, MAPPING)
    assert got["c"]["buckets"] == R.as_json(R.page(docs, spec), spec)
    ctx.unregister_split("comp-wide")
