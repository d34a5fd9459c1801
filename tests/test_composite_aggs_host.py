"""Composite aggregations on the host (no GPU): request parsing and its refusals, the lowering to a chain of source
nodes with the per-split `after` bound the walk filters with, and entries -> intermediate -> merge -> finalize against
composite_ref's brute force, including both REST goldens and after_key paging."""
import json

import numpy as np
import pytest

from quickwit_b200 import ffi, proto, service, splitgen as S
import composite_ref as R
import pipeline as PL
from test_oracle_goldens import AGG_MAPPING, AGG_SPLIT1, AGG_SPLIT2

GOLDEN = {"size": 5, "sources": [{"host": {"terms": {"field": "host", "missing_bucket": True}}},
                                 {"name": {"terms": {"field": "name"}}},
                                 {"response": {"histogram": {"field": "response", "interval": 50}}}]}
GOLDEN_AFTER = {"host": "str:192.168.0.10", "name": "str:Albert", "response": "f64:100"}


@pytest.fixture(scope="module")
def golden_splits():
    return [(S.build_split(AGG_SPLIT1, AGG_MAPPING, "agg-1"), AGG_SPLIT1), (S.build_split(AGG_SPLIT2, AGG_MAPPING, "agg-2"), AGG_SPLIT2)]


def _plan(img, spec, mapping=AGG_MAPPING, name="c"):
    req = PL.search_request(PL.MATCH_ALL, max_hits=0, aggs={name: {"composite": spec}})
    return req, service.compile_plan(img, req, json.dumps(mapping))


def _nodes(plan):
    h = ffi.QwPlanHeader.from_buffer_copy(plan)
    off = ffi.C.sizeof(ffi.QwPlanHeader) + h.num_nodes * ffi.C.sizeof(ffi.QwPlanNode)
    return [ffi.QwAggNode.from_buffer_copy(plan, off + i * ffi.C.sizeof(ffi.QwAggNode)) for i in range(h.num_aggs)]


def _search(splits, spec, mapping=AGG_MAPPING):
    """entries of every split (brute force) -> leaf responses -> leaf merge -> finalize"""
    aggs = {"c": {"composite": spec}}
    req = PL.search_request(PL.MATCH_ALL, max_hits=0, aggs=aggs)
    dm = json.dumps(mapping)
    parts = []
    for img, docs in splits:
        plan = service.compile_plan(img, req, dm)
        parts.append(service.build_leaf_response_entries(img, req, dm, len(docs), [], R.split_entries(img, plan, docs, spec)))
    merged = proto.dec_leaf_search_response(service.merge_leaf_responses(req, parts))
    return json.loads(service.finalize_aggregation(json.dumps(aggs), merged["intermediate_aggregation_result"] or b""))["c"]


def test_rest_goldens(golden_splits):
    got = _search(golden_splits, GOLDEN)
    assert got["buckets"] == [
        {"key": {"host": None, "name": "Bernhard", "response": 100.0}, "doc_count": 1},
        {"key": {"host": None, "name": "Fritz", "response": 0.0}, "doc_count": 2},
        {"key": {"host": "192.168.0.1", "name": "Fred", "response": 100.0}, "doc_count": 1},
        {"key": {"host": "192.168.0.1", "name": "Fritz", "response": 0.0}, "doc_count": 1},
        {"key": {"host": "192.168.0.10", "name": "Albert", "response": 100.0}, "doc_count": 1}]
    assert got["after_key"] == GOLDEN_AFTER
    nxt = _search(golden_splits, dict(GOLDEN, after=got["after_key"]))
    assert nxt["buckets"] == [
        {"key": {"host": "192.168.0.10", "name": "Holger", "response": 0.0}, "doc_count": 1},
        {"key": {"host": "192.168.0.10", "name": "Werner", "response": 0.0}, "doc_count": 1},
        {"key": {"host": "192.168.0.11", "name": "Manfred", "response": 100.0}, "doc_count": 1}]
    assert nxt["after_key"] == {"host": "str:192.168.0.11", "name": "str:Manfred", "response": "f64:100"}
    # plain after values page the same way; past the last bucket: no buckets, after_key {}
    plain = _search(golden_splits, dict(GOLDEN, after={"host": "192.168.0.10", "name": "Albert", "response": 100}))
    assert plain == nxt
    assert _search(golden_splits, dict(GOLDEN, after=nxt["after_key"])) == {"after_key": {}, "buckets": []}


@pytest.mark.parametrize("size", [1, 2, 3, 7])
@pytest.mark.parametrize("orders", [("asc", "asc", "asc"), ("desc", "asc", "desc"), ("desc", "desc", "desc")])
def test_paging_to_exhaustion_equals_brute_force(golden_splits, size, orders):
    spec = {"size": size, "sources": [{"host": {"terms": {"field": "host", "missing_bucket": True, "order": orders[0]}}},
                                      {"resp": {"histogram": {"field": "response", "interval": 25, "missing_bucket": True, "order": orders[1]}}},
                                      {"name": {"terms": {"field": "name", "order": orders[2]}}}]}
    want = R.as_json(R.all_buckets(AGG_SPLIT1 + AGG_SPLIT2, spec), spec)
    got, after = [], None
    for _ in range(len(want) + 1):
        page = _search(golden_splits, spec if after is None else dict(spec, after=after))
        got += page["buckets"]
        if not page["buckets"]:
            assert page["after_key"] == {}
            break
        after = page["after_key"]
    assert got == want


def _random_splits(n_splits, seed):
    rng = np.random.default_rng(seed)
    mapping = {"field_mappings": [{"name": "svc", "type": "text", "tokenizer": "raw", "fast": True},
                                  {"name": "tags", "type": "u64", "fast": True},
                                  {"name": "code", "type": "i64", "fast": True},
                                  {"name": "lat", "type": "f64", "fast": True}]}
    out = []
    for s in range(n_splits):
        docs = []
        for _ in range(int(rng.integers(40, 120))):
            d = {"code": int(rng.integers(-20, 20)), "lat": float(rng.integers(0, 400)) / 4}
            if rng.random() < 0.8:
                d["svc"] = f"s{int(rng.integers(0, 9))}"
            k = int(rng.integers(0, 3))
            if k:
                d["tags"] = sorted({int(x) for x in rng.integers(0, 6, size=k)})
            docs.append(d)
        out.append((S.build_split(docs, mapping, f"rnd-{seed}-{s}"), docs))
    return out, mapping


@pytest.mark.parametrize("seed", [1, 2])
def test_merge_of_three_splits_equals_brute_force(seed):
    splits, mapping = _random_splits(3, seed)
    docs = [d for _img, ds in splits for d in ds]
    spec = {"size": 9, "sources": [{"svc": {"terms": {"field": "svc", "missing_bucket": True}}},
                                   {"tags": {"terms": {"field": "tags", "missing_bucket": True, "order": "desc"}}},
                                   {"lat": {"histogram": {"field": "lat", "interval": 20}}}]}
    want_all = R.as_json(R.all_buckets(docs, spec), spec)
    pos = 0
    after = None
    while True:
        page = _search(splits, spec if after is None else dict(spec, after=after), mapping)
        assert page["buckets"] == want_all[pos:pos + 9]
        pos += len(page["buckets"])
        if not page["buckets"]:
            break
        after = page["after_key"]
    assert pos == len(want_all)


# ---- parsing and refusals ---------------------------------------------------------------------------------------------
def _code(img, spec=None, aggs=None):
    aggs = aggs if aggs is not None else {"c": {"composite": spec}}
    with pytest.raises(ffi.QwGpuError) as e:
        service.compile_plan(img, PL.search_request(PL.MATCH_ALL, max_hits=0, aggs=aggs), json.dumps(AGG_MAPPING))
    return e.value.code


def test_refusals(golden_splits):
    img = golden_splits[0][0]
    src = [{"h": {"terms": {"field": "host"}}}]
    inv, uns = ffi.EINVALID_AGG, ffi.EUNSUPPORTED
    assert _code(img, {}) == inv
    assert _code(img, {"sources": []}) == inv
    assert _code(img, {"sources": src + src}) == inv
    assert _code(img, {"sources": [{"h": {"range": {"field": "host"}}}]}) == inv
    assert _code(img, {"sources": src, "size": 0}) == inv
    assert _code(img, {"sources": src, "after": {}}) == inv
    assert _code(img, {"sources": src, "after": {"h": "a", "x": "b"}}) == inv
    assert _code(img, {"sources": [{"r": {"histogram": {"field": "response", "interval": 5}}}], "after": {"r": "str:x"}}) == inv
    assert _code(img, {"sources": src, "after": {"h": None}}) == inv  # null without missing_bucket
    assert _code(img, {"sources": src, "after": {"h": "u64:-1"}}) == inv
    assert _code(img, aggs={"t": {"terms": {"field": "host"}, "aggs": {"c": {"composite": {"sources": src}}}}}) == uns
    for k, v in (("missing_order", "first"), ("format", "x"), ("script", "x")):
        assert _code(img, {"sources": [{"h": {"terms": {"field": "host", k: v}}}]}) == uns
    assert _code(img, {"sources": [{"d": {"date_histogram": {"field": "date", "calendar_interval": "1d"}}}]}) == uns
    assert _code(img, {"sources": src, "size": 65001}) == uns
    _plan(img, {"sources": src, "size": 65000})
    # n sources take n nodes: 8 fit a plan, 9 do not (refused when the plan is lowered for the GPU)
    nine = [{f"s{i}": {"terms": {"field": "host"}}} for i in range(9)]
    assert len(_nodes(_plan(img, {"sources": nine})[1])) == 9


# ---- lowering and the per-split after bound ---------------------------------------------------------------------------
def test_chain_lowering(golden_splits):
    img = golden_splits[0][0]
    req = PL.search_request(PL.MATCH_ALL, max_hits=0, aggs={"c": {"composite": GOLDEN, "aggs": {"a": {"avg": {"field": "response"}}}},
                                                            "t": {"terms": {"field": "name"}}})
    plan = service.compile_plan(img, req, json.dumps(AGG_MAPPING))
    n = _nodes(plan)
    assert [x.kind for x in n] == [ffi.AGG_TERMS, ffi.AGG_TERMS, ffi.AGG_TERMS, ffi.AGG_HISTOGRAM, ffi.AGG_STATS]
    assert (n[0].first_child, n[0].num_children, n[2].first_child, n[3].first_child, n[3].num_children) == (2, 1, 3, 4, 1)
    assert [x.reserved for x in n] == [ffi.AGG_COMP_LEVEL | ffi.AGG_COMP_MISSING, 0, ffi.AGG_COMP_LEVEL,
                                       ffi.AGG_COMP_LEVEL | ffi.AGG_COMP_LAST, 0]
    assert n[0].range_to[0] == 5 and n[0].has_missing == 1
    assert service.agg_layout(img, plan)[0]


def _bound(img, src, after, mapping=AGG_MAPPING):
    n = _nodes(_plan(img, {"sources": [src], "after": after}, mapping)[1])[0]
    return n.range_from[0], n.reserved & ~(ffi.AGG_COMP_LEVEL | ffi.AGG_COMP_LAST | ffi.AGG_COMP_MISSING | ffi.AGG_COMP_DESC)


def test_after_bound(golden_splits):
    img = golden_splits[0][0]
    HA, EX, NUL, ALL = ffi.AGG_COMP_HAS_AFTER, ffi.AGG_COMP_EXACT, ffi.AGG_COMP_AFTER_NULL, ffi.AGG_COMP_AFTER_ALL
    hosts = sorted({d["host"] for d in AGG_SPLIT1})
    h = {"h": {"terms": {"field": "host", "missing_bucket": True}}}
    hd = {"h": {"terms": {"field": "host", "missing_bucket": True, "order": "desc"}}}
    assert _bound(img, h, {"h": "str:192.168.0.10"}) == (hosts.index("192.168.0.10"), HA | EX)
    assert _bound(img, h, {"h": "192.168.0.100"}) == (hosts.index("192.168.0.11"), HA)  # between two terms
    assert _bound(img, hd, {"h": "192.168.0.100"}) == (hosts.index("192.168.0.10"), HA)
    assert _bound(img, h, {"h": "3"})[1] == HA | ALL
    assert _bound(img, hd, {"h": "0"})[1] == HA | ALL
    assert _bound(img, h, {"h": None}) == (0, HA | NUL)
    # an after value whose type the source's column cannot hold is refused
    for bad in (5, "bool:true", True, "f64:1.5"):
        assert _code(img, {"sources": [h], "after": {"h": bad}}) == ffi.EINVALID_AGG
    for bad in ("str:100", "x", "bool:false"):
        assert _code(img, {"sources": [{"r": {"terms": {"field": "response"}}}], "after": {"r": bad}}) == ffi.EINVALID_AGG
    # numbers: response holds 30, 100, 100, 120 (raw = (v - 30) / gcd 10)
    r = {"r": {"terms": {"field": "response"}}}
    rd = {"r": {"terms": {"field": "response", "order": "desc"}}}
    assert _bound(img, r, {"r": 100}) == (7, HA | EX)
    assert _bound(img, r, {"r": 101}) == (8, HA)
    assert _bound(img, r, {"r": 100.5}) == (8, HA)
    assert _bound(img, rd, {"r": 101}) == (7, HA)
    assert _bound(img, r, {"r": -5}) == (0, HA)
    assert _bound(img, r, {"r": 121})[1] == HA | ALL
    assert _bound(img, rd, {"r": 29})[1] == HA | ALL
    assert _bound(img, rd, {"r": 10 ** 6}) == (9, HA)
    # histogram: interval 50 from position 0 (0, 50, 100)
    hh = {"r": {"histogram": {"field": "response", "interval": 50}}}
    hhd = {"r": {"histogram": {"field": "response", "interval": 50, "order": "desc"}}}
    assert _bound(img, hh, {"r": "f64:100"}) == (2, HA | EX)
    assert _bound(img, hh, {"r": 60}) == (2, HA)
    assert _bound(img, hhd, {"r": 60}) == (1, HA)
    assert _bound(img, hh, {"r": -1}) == (0, HA)
    assert _bound(img, hh, {"r": 101})[1] == HA | ALL


def test_after_key_formatting(golden_splits):
    spec = {"size": 1, "sources": [{"r": {"histogram": {"field": "response", "interval": 0.1}}}]}
    got = _search(golden_splits[:1], spec)
    assert got["after_key"] == {"r": "f64:30"}
    spec = {"size": 1, "sources": [{"r": {"terms": {"field": "response"}}}]}
    assert _search(golden_splits[:1], dict(spec, after={"r": 30}))["after_key"] in ({"r": "i64:100"}, {"r": "u64:100"})


def test_histogram_bound_with_an_offset_far_larger_than_the_interval(golden_splits):
    """Neighbouring positions round to one key in f64: the lowering gives up the device filter (and the device cut)
    after a few correction steps instead of walking ulp(offset) / interval positions."""
    import time
    img = golden_splits[0][0]
    for off in (1e24, 1e26, 1e30, 1e300):
        src = {"r": {"histogram": {"field": "response", "interval": 1, "offset": off}}}
        t0 = time.monotonic()
        bound, flags = _bound(img, src, {"r": off})
        assert time.monotonic() - t0 < 1.0
        assert flags & ffi.AGG_COMP_AFTER_HOST and not flags & ffi.AGG_COMP_HAS_AFTER
    dh = {"d": {"date_histogram": {"field": "date", "fixed_interval": "1s", "offset": "900000000000000000000s"}}}
    assert _bound(img, dh, {"d": 9e23})[1] & ffi.AGG_COMP_AFTER_HOST
