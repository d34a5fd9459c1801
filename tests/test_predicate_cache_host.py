"""QueryAst `cache` nodes through the plan compiler, on the CPU:
  * in a request that reads no scores, `cache` compiles to a QW_NODE_CACHE whose subtree is exactly the plan nodes of
    its inner query compiled alone (compared in the engine's cache-key form: breadth-first, children rebased, boost and
    bm25_weight zeroed);
  * in a request ranked by _score, the plan bytes equal those of the inner query alone;
  * the [start_timestamp, end_timestamp) filter stays outside the node.
`strip` turns a plan with CACHE nodes into the plan without them (each node replaced by its child): the oracle and the
GPU module compare results against it."""
from __future__ import annotations

import ctypes as C
import json
import random
from typing import List, Tuple

import pytest

from hypothesis import HealthCheck, given, settings, strategies as st

from quickwit_b200 import ffi, plan as P, proto, service, splitgen as S
from helpers import assert_same
from regex_ref import oracle_search
import test_gpu_fuzz as _F  # (its generator; its own tests need a GPU)

SYNTH_MAPPING = {"field_mappings": [{"name": "body", "type": "text", "record": "freq", "fieldnorms": True},
                                    {"name": "severity_text", "type": "text", "tokenizer": "raw", "fast": True},
                                    {"name": "timestamp", "type": "datetime", "fast": True, "fast_precision": "seconds"},
                                    {"name": "tenant_id", "type": "u64", "fast": True},
                                    {"name": "msg", "type": "text", "record": "position", "fieldnorms": True}],
                 "timestamp_field": "timestamp"}
DM = json.dumps(SYNTH_MAPPING)
HDR, NODE = C.sizeof(ffi.QwPlanHeader), C.sizeof(ffi.QwPlanNode)
PARENTS = (ffi.NODE_BOOL, ffi.NODE_PHRASE, ffi.NODE_PHRASE_PREFIX, ffi.NODE_TERM_SET, ffi.NODE_CACHE)


def cache(q):
    return {"type": "cache", "inner": q}


def term(field, value):
    return {"type": "term", "field": field, "value": value}


def phrase(text):
    return {"type": "full_text", "field": "msg", "text": text, "params": {"mode": {"type": "phrase"}}}


def regex(r):
    return {"type": "regex", "field": "msg", "regex": r}


def tenant_range(lo, hi):
    return {"type": "range", "field": "tenant_id", "lower_bound": {"Included": lo}, "upper_bound": {"Excluded": hi}}


INNER = {
    "term": term("body", "t1"),
    "phrase": phrase("w1 w2"),
    "long phrase": phrase("w1 w2 w3 w4 w5 w6 w7 w8 w9 w10"),
    "regex": regex("w1.*"),
    "range": tenant_range(10, 60),
    "bool": {"type": "bool", "must": [term("body", "t0")], "should": [term("body", "t2"), phrase("w3 w4")],
             "must_not": [term("body", "t3")], "filter": [tenant_range(0, 80)]},
}


def parse(plan: bytes) -> Tuple[ffi.QwPlanHeader, List[ffi.QwPlanNode]]:
    h = ffi.QwPlanHeader.from_buffer_copy(plan[:HDR])
    nodes = [ffi.QwPlanNode.from_buffer_copy(plan[HDR + i * NODE:HDR + (i + 1) * NODE]) for i in range(h.num_nodes)]
    return h, nodes


def canon(nodes: List[ffi.QwPlanNode], root: int) -> bytes:
    """The engine's cache key of the subtree at `root` (engine.cu pred_key), restated."""
    out = [ffi.QwPlanNode.from_buffer_copy(bytes(nodes[root]))]
    i = 0
    while i < len(out):
        n = out[i]
        n.boost = n.bm25_weight = 0.0
        if n.kind not in PARENTS or not n.num_children:
            n.first_child = n.num_children = 0
        else:
            first, cnt = n.first_child, n.num_children
            n.first_child = len(out)
            out.extend(ffi.QwPlanNode.from_buffer_copy(bytes(nodes[first + k])) for k in range(cnt))
        i += 1
    out[0].occur = ffi.OCCUR_MUST
    return b"".join(bytes(n) for n in out)


def strip(plan: bytes) -> bytes:
    """The plan with every CACHE node replaced by its child (in the node's own clause position)."""
    h, nodes = parse(plan)
    changed = True
    while changed:
        changed = False
        for n in nodes:
            if n.kind == ffi.NODE_CACHE:
                occur = n.occur
                C.memmove(C.addressof(n), C.addressof(nodes[n.first_child]), NODE)
                n.occur = occur
                changed = True
    return plan[:HDR] + b"".join(bytes(n) for n in nodes) + plan[HDR + h.num_nodes * NODE:]


def cache_nodes(plan: bytes) -> List[int]:
    return [i for i, n in enumerate(parse(plan)[1]) if n.kind == ffi.NODE_CACHE]


def compile_(img, q, **kw) -> bytes:
    return service.compile_plan(img, proto.enc_search_request(json.dumps(q), **kw), DM)


@pytest.fixture(scope="module")
def img():
    return S.synth_split(6000, 0, [0.2, 0.1, 0.05, 0.01], split_id="pc-host", msg_vocab=64)


UNSCORED = dict(max_hits=10, sort_fields=[("timestamp", 1)])
SCORED = dict(max_hits=10, sort_fields=[("_score", 1)])


def placements(inner):
    """(label, query with the cached inner query, path of the CACHE node's expected occur)"""
    other = term("body", "t0")
    return [
        ("root", cache(inner), ffi.OCCUR_MUST),
        ("must", {"type": "bool", "must": [cache(inner), other]}, ffi.OCCUR_MUST),
        ("filter", {"type": "bool", "must": [other], "filter": [cache(inner)]}, ffi.OCCUR_FILTER),
        ("should", {"type": "bool", "should": [cache(inner), other]}, ffi.OCCUR_SHOULD),
        ("must_not", {"type": "bool", "must": [other], "must_not": [cache(inner)]}, ffi.OCCUR_MUST_NOT),
        ("nested", {"type": "bool", "must": [other], "filter": [cache({"type": "bool", "must": [cache(inner), term("body", "t2")]})]},
         ffi.OCCUR_FILTER),
    ]


def uncache(q):
    if isinstance(q, dict):
        if q.get("type") == "cache":
            return uncache(q["inner"])
        return {k: uncache(v) for k, v in q.items()}
    if isinstance(q, list):
        return [uncache(x) for x in q]
    return q


@pytest.mark.parametrize("name", list(INNER))
def test_unscored_cache_is_the_inner_plan(img, name):
    inner = INNER[name]
    want = canon(parse(compile_(img, inner, **UNSCORED))[1], 0)
    for label, q, occur in placements(inner):
        plan = compile_(img, q, **UNSCORED)
        _, nodes = parse(plan)
        idx = cache_nodes(plan)
        assert len(idx) == (2 if label == "nested" else 1), label
        assert nodes[idx[0]].occur == occur and all(nodes[i].num_children == 1 for i in idx), label
        # the innermost CACHE node holds exactly the plan nodes of the inner query compiled alone
        assert [canon(nodes, nodes[i].first_child) == want for i in idx].count(True) == 1, label
        # with the CACHE nodes replaced by their children, the plan is the query's without them (except where
        # simplify would flatten a cached bool into its parent: the node is opaque to it)
        if label != "nested":
            assert canon(parse(strip(plan))[1], 0) == canon(parse(compile_(img, uncache(q), **UNSCORED))[1], 0), label


@pytest.mark.parametrize("name", [n for n in INNER if n != "regex"])  # (a regex is refused in a scoring clause)
def test_scored_cache_compiles_the_inner_query(img, name):
    for label, q, _ in placements(INNER[name]):
        assert compile_(img, q, **SCORED) == compile_(img, uncache(q), **SCORED), label


def test_timestamp_filter_stays_outside(img):
    ts = dict(UNSCORED, start_timestamp=1_700_000_000 + 3_600, end_timestamp=1_700_000_000 + 40_000)
    plan = compile_(img, cache(INNER["bool"]), **ts)
    _, nodes = parse(plan)
    ts_col = img.column_ord("timestamp")
    assert nodes[0].kind == ffi.NODE_BOOL
    kids = [nodes[nodes[0].first_child + k] for k in range(nodes[0].num_children)]
    assert [(k.kind, k.occur) for k in kids] == [(ffi.NODE_CACHE, ffi.OCCUR_MUST), (ffi.NODE_RANGE, ffi.OCCUR_FILTER)]
    assert kids[1].column == ts_col
    sub = canon(nodes, kids[0].first_child)
    assert sub == canon(parse(compile_(img, INNER["bool"], **UNSCORED))[1], 0)
    assert all(ffi.QwPlanNode.from_buffer_copy(sub[i:i + NODE]).column != ts_col for i in range(0, len(sub), NODE))


def test_count_only_request_caches(img):
    """max_hits 0 clears the sort: nothing reads scores, even for a _score sort."""
    plan = compile_(img, cache(INNER["term"]), max_hits=0, sort_fields=[("_score", 1)])
    assert parse(plan)[1][0].kind == ffi.NODE_CACHE


def test_cache_without_inner_is_refused(img):
    with pytest.raises(ffi.QwGpuError):
        compile_(img, {"type": "cache"}, **UNSCORED)


# ---- the fuzz generator's bool trees x sort specs ------------------------------------------------------------------
def with_cache(root: "P.Node", seed: int) -> "P.Node":
    """`root` with CACHE nodes around a random third of its clauses (and sometimes around the root), nested ones
    included; the nodes keep their clause's occur."""
    rnd = random.Random(seed)
    def walk(n):
        kids = [walk(c) for c in n.children] if n.kind == ffi.NODE_BOOL else n.children
        m = P.Node(n.kind, n.occur, n.boost, children=kids, min_should_match=n.msm, term_ord=n.term_ord,
                   field_id=n.field_id, weight=n.weight, column=n.column, lo=n.lo, hi=n.hi)
        return P.cache(m) if rnd.random() < 0.33 else m
    return walk(root)


@pytest.fixture(scope="module")
def fuzz_img():
    return _F._clustered_split("pc-fuzz-host")


@settings(max_examples=60, deadline=None, derandomize=True, suppress_health_check=list(HealthCheck))
@given(kids=_F._tree(), msm=st.sampled_from([None, None, 1, 2]), sort=_F._SORTS, k=st.sampled_from([0, 7, 100, 1000]),
       with_aggs=st.integers(0, 2), seed=st.integers(0, 1 << 30))
def test_fuzz_cache_as_its_child(fuzz_img, kids, msm, sort, k, with_aggs, seed):
    """The oracle's hits, counts and aggregation cells for each fuzz plan with CACHE nodes (each evaluated as its child,
    `strip`) equal those of the plan without them."""
    F, img = _F, fuzz_img
    aggs = [F.terms_agg(img, "code"), F.histogram_agg(img, "timestamp", 3600e9)] if with_aggs == 1 else \
        [F.terms_agg(img, "code", children=[F.stats_agg(img, "timestamp")])] if with_aggs == 2 else []
    root = F._build(img, kids, msm=msm)
    plain = P.make_plan(root, k, F._sort(img, sort), aggs=aggs)
    cached = P.make_plan(with_cache(root, seed), k, F._sort(img, sort), aggs=aggs)
    assert cache_nodes(cached) or not cache_nodes(plain)
    assert_same(oracle_search(img, strip(cached)), oracle_search(img, plain), ctx=f"kids={kids} sort={sort} k={k} seed={seed}")
