"""Aggregation plans of 9 to 32 nodes on the host: compiled requests of 9, 16 and 32 nodes have the intended tree and
layout; the CPU oracle agrees with the brute force on every plan test_gpu_wide_aggs.py runs; the restatement of
k_aggscan's eligibility takes 8 flat nodes and leaves 9 to k_window; and a 32-node request merged over three splits and
finalised equals a JSON brute force computed from the documents."""
import json

import pytest

from quickwit_b200 import ffi, plan as P, service
from oracle import oracle as O
from agg_ref import _layout, assert_cells, cells
import percentiles_ref as PR
import pipeline as PL
import wide_aggs_cases as W


@pytest.fixture(scope="module")
def split():
    return W.WideSplit("wide-host", W.make_docs(3001, 1))


def test_limits_exported():
    assert (ffi.MAX_AGG_NODES, ffi.MAX_AGG_LEVELS, ffi.MAX_AGG_COLUMNS) == (W.MAX_NODES, W.MAX_LEVELS, W.MAX_AGG_COLUMNS)
    header = open(__file__.rsplit("/tests/", 1)[0] + "/include/qwgpu.h").read()
    for name, v in (("NODES", 32), ("LEVELS", 8), ("COLUMNS", 32)):
        assert f"#define QWGPU_MAX_AGG_{name} {v}u" in header


# ---- compiled requests -----------------------------------------------------------------------------------------------
def _request(n, levels):
    """A JSON aggregation request of exactly n nodes: terms / histogram / range / metric nodes, nested `levels` deep."""
    metrics = [{"avg": {"field": "lat"}}, {"max": {"field": "code"}}, {"stats": {"field": "latf"}},
               {"value_count": {"field": "lvl"}}, {"sum": {"field": "opt"}}]
    buckets = [{"terms": {"field": "svc"}}, {"histogram": {"field": "lat", "interval": 500}},
               {"range": {"field": "code", "ranges": [{"to": 0}, {"from": 0}]}}, {"terms": {"field": "tags"}}]
    out, left, i = {}, n, 0
    while left:
        if levels > 1 and left >= levels:
            node = dict(buckets[i % len(buckets)])
            cur, left = node, left - 1
            for d in range(1, levels):
                last = d == levels - 1
                child = dict(metrics[(i + d) % len(metrics)] if last else buckets[(i + d) % len(buckets)])
                cur["aggs"] = {f"n{i}_{d}": child}
                cur, left = child, left - 1
            out[f"n{i}"] = node
        else:
            out[f"n{i}"] = dict(metrics[i % len(metrics)] if i % 2 else buckets[i % len(buckets)])
            left -= 1
        i += 1
    return out


@pytest.mark.parametrize("levels", [1, 3, 8])
@pytest.mark.parametrize("n", [9, 16, 32])
def test_compiled_shape(split, n, levels):
    req = PL.search_request(PL.MATCH_ALL, max_hits=0, aggs=_request(n, levels))
    plan = service.compile_plan(split.img, req, json.dumps(W.MAPPING))
    nodes = PR.plan_nodes(plan)
    assert len(nodes) == n
    depth = 0
    for i, g in enumerate(nodes):
        for c in range(g.first_child, g.first_child + g.num_children):
            assert nodes[c].parent == i
        d, p = 1, g.parent
        while p != ffi.ABSENT:
            assert p < i  # parents come first (breadth-first order)
            d, p = d + 1, nodes[p].parent
        depth = max(depth, d)
    assert depth == levels
    hashed, _bound = service.agg_layout(split.img, plan)
    assert bool(hashed) == (levels > 3)  # bucket > bucket > metric is the deepest dense tree


# ---- oracle against the brute force on the GPU test's plans ------------------------------------------------------------
def _check_oracle(sp, aggs, root=None, max_hits=0, sort=((ffi.SORT_DOCID, ffi.ORDER_DESC, ffi.ABSENT),), docs=None):
    plan = P.make_plan(root or P.bool_([P.match_all()]), max_hits, sort, aggs=aggs)
    assert_cells(O.split_search(sp.img, plan).cells, cells(aggs, sp.cols, docs), f"{W.count_nodes(aggs)} nodes")


@pytest.mark.parametrize("levels", [1, 2, 3])
@pytest.mark.parametrize("n", [9, 16, 32])
def test_oracle_dense(split, n, levels):
    aggs = W.dense_tree(split, n, levels)
    assert W.count_nodes(aggs) == n and not service.agg_layout(split.img, P.make_plan(P.match_all(), 0, aggs=aggs))[0]
    _check_oracle(split, aggs)
    docs = [i for i, d in enumerate(split.docs) if "b" in d["body"].split()]
    _check_oracle(split, aggs, P.bool_([P.term(split.img, "body", "b")]), 10, ((ffi.SORT_SCORE, ffi.ORDER_DESC, ffi.ABSENT),), docs)


@pytest.mark.parametrize("n", [9, 17, 32])
def test_oracle_fast_plans(split, n):
    aggs = W.fast_plan(split, n)
    assert W.count_nodes(aggs) == n and sum(x for *_a, x in _layout(aggs)) <= W.QA_MAX_CELLS
    _check_oracle(split, aggs)


@pytest.mark.parametrize("n", [9, 32])
def test_oracle_hashed_trees(split, n):
    aggs = W.hashed_tree(split, n)
    assert W.depth_of(aggs) == W.MAX_LEVELS and service.agg_layout(split.img, P.make_plan(P.match_all(), 0, aggs=aggs))[0]
    _check_oracle(split, aggs)


def test_oracle_flat_aggscan_plans(split):
    for n in (8, 9):
        _check_oracle(split, W.aggscan_flat(split, n))


# ---- k_aggscan's eligibility -----------------------------------------------------------------------------------------
def test_aggscan_eligibility(split):
    def eligible(aggs, query_all=True, max_hits=0):
        n_cells = sum(x for *_a, x in _layout(aggs))
        hdr = split.img.columns()
        full32 = all(hdr[a.column].cardinality == ffi.CARD_FULL and hdr[a.column].bits <= 32 for a in aggs)
        return W.aggscan_eligible(aggs, n_cells, query_all, max_hits, full32)

    assert eligible(W.aggscan_flat(split, 1)) and eligible(W.aggscan_flat(split, 8))
    assert not eligible(W.aggscan_flat(split, 9)) and not eligible(W.aggscan_flat(split, 32))
    assert not eligible(W.aggscan_flat(split, 8), max_hits=1) and not eligible(W.aggscan_flat(split, 8), query_all=False)
    assert not eligible(W.fast_plan(split, 9)[:1])  # stats children
    assert not eligible([split.terms("lvl")])      # a multi-valued column


# ---- a 32-node request over three splits, finalised, against a JSON brute force -----------------------------------------
def _vals(d, f):
    v = d.get(f)
    return [] if v is None else (v if isinstance(v, list) else [v])


def _metric_json(kind, vals):
    vals = [float(v) for v in vals]
    s = float(sum(vals))
    if kind == "stats":
        return {"count": len(vals), "sum": s, "min": min(vals) if vals else None, "max": max(vals) if vals else None,
                "avg": s / len(vals) if vals else None}
    return {"value": {"avg": s / len(vals) if vals else None, "sum": s, "min": min(vals) if vals else None,
                      "max": max(vals) if vals else None, "value_count": float(len(vals))}[kind]}


def brute_json(aggs, docs):
    """Finalised JSON of terms (single-valued fields, at most `size` keys: no cut), gap-free histograms and the
    metrics, from the documents."""
    out = {}
    for name, spec in aggs.items():
        kind = next(k for k in spec if k != "aggs")
        p, subs = spec[kind], spec.get("aggs", {})
        if kind == "terms":
            groups = {}
            for d in docs:
                for v in set(_vals(d, p["field"])):
                    groups.setdefault(v, []).append(d)
            keys = sorted(groups, key=lambda k: (-len(groups[k]), k))
            assert len(keys) <= p.get("size", 10)
            out[name] = {"buckets": [{"key": k, "doc_count": len(groups[k]), **brute_json(subs, groups[k])} for k in keys],
                         "doc_count_error_upper_bound": 0, "sum_other_doc_count": 0}
        elif kind == "histogram":
            iv, groups = p["interval"], {}
            for d in docs:
                for v in _vals(d, p["field"]):
                    groups.setdefault(float(v // iv * iv), []).append(d)
            keys = sorted(groups)
            assert len(keys) == int((keys[-1] - keys[0]) / iv) + 1  # no empty bucket in between
            out[name] = {"buckets": [{"key": k, "doc_count": len(groups[k]), **brute_json(subs, groups[k])} for k in keys]}
        else:
            out[name] = _metric_json(kind, [v for d in docs for v in _vals(d, p["field"])])
    return out


WIDE32 = {
    "by_svc": {"terms": {"field": "svc"}, "aggs": {
        "lat_avg": {"avg": {"field": "lat"}}, "code_min": {"min": {"field": "code"}}, "code_max": {"max": {"field": "code"}},
        "lat_stats": {"stats": {"field": "lat"}}, "k00_sum": {"sum": {"field": "k00"}}, "lvl_count": {"value_count": {"field": "lvl"}}}},
    "by_lat": {"histogram": {"field": "lat", "interval": 1000}, "aggs": {
        "code_avg": {"avg": {"field": "code"}}, "lat_sum": {"sum": {"field": "lat"}}, "k01_max": {"max": {"field": "k01"}}}},
    "by_k02": {"terms": {"field": "k02"}, "aggs": {
        "code_stats": {"stats": {"field": "code"}}, "k03_avg": {"avg": {"field": "k03"}},
        "by_k04": {"terms": {"field": "k04"}, "aggs": {"lat_sum": {"sum": {"field": "lat"}}, "lat_min": {"min": {"field": "lat"}}}}}},
    "lat_avg": {"avg": {"field": "lat"}}, "code_sum": {"sum": {"field": "code"}}, "lat_min": {"min": {"field": "lat"}},
    "lat_max": {"max": {"field": "lat"}}, "code_stats": {"stats": {"field": "code"}}, "tags_count": {"value_count": {"field": "tags"}},
    "k05_avg": {"avg": {"field": "k05"}}, "k06_sum": {"sum": {"field": "k06"}}, "k07_stats": {"stats": {"field": "k07"}},
    "by_k08": {"terms": {"field": "k08"}, "aggs": {
        "lat_avg": {"avg": {"field": "lat"}},
        "by_code": {"histogram": {"field": "code", "interval": 25}, "aggs": {
            "lvl_count": {"value_count": {"field": "lvl"}}, "lat_max": {"max": {"field": "lat"}}}}}},
    "k09_max": {"max": {"field": "k09"}}}


def test_32_nodes_merged_and_finalised():
    splits = [W.WideSplit(f"wide-json-{i}", W.make_docs(n, 70 + i)) for i, n in enumerate((1500, 777, 2100))]
    req = PL.search_request(PL.MATCH_ALL, max_hits=0, aggs=WIDE32)
    plan = service.compile_plan(splits[0].img, req, json.dumps(W.MAPPING))
    assert len(PR.plan_nodes(plan)) == 32
    got = PL.cpu_root_search([sp.img for sp in splits], PL.MATCH_ALL, W.MAPPING, max_hits=0, aggs=WIDE32)["aggregations"]
    assert got == brute_json(WIDE32, [d for sp in splits for d in sp.docs])
