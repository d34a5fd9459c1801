"""The partial-result cache on the GPU (LeafSearchCache, quickwit-search/src/leaf_cache.rs; DESIGN.md §7.1).

A response served with the cache on must equal the response of the same call with the cache off in everything but
`resource_stats`: hits, num_hits, the finalized aggregations, failed_splits and the split counters. Over 32 splits
with day-long time ranges, a dashboard window of eight days slides by one day: the splits it covers in both positions
hit, the splits at its edges miss. Every test here turns the cache on for the shared context and off again."""
import json
import os
import subprocess
import sys
import textwrap
from concurrent.futures import ThreadPoolExecutor

import pytest

from quickwit_b200 import proto, service, splitgen as S
from quickwit_b200.service import SearcherContext

pytestmark = pytest.mark.gpu

T0 = 1_700_000_000
DAY = 86_400
N_SPLITS = 32
FRACS = [0.2, 0.1, 0.05, 0.02, 0.01]
MAPPING = {"field_mappings": [{"name": "body", "type": "text", "record": "freq", "fieldnorms": True},
                              {"name": "severity_text", "type": "text", "tokenizer": "raw", "fast": True},
                              {"name": "timestamp", "type": "datetime", "fast": True, "fast_precision": "seconds"},
                              {"name": "tenant_id", "type": "u64", "fast": True}], "timestamp_field": "timestamp"}
DM = json.dumps(MAPPING)
BUDGET = 64 << 20


def term(v):
    return {"type": "term", "field": "body", "value": v}


OR4 = {"type": "bool", "should": [term(f"t{i}") for i in range(4)]}
TERMS_HIST_AVG = {"sev": {"terms": {"field": "severity_text"},
                          "aggs": {"h": {"date_histogram": {"field": "timestamp", "fixed_interval": "1h"},
                                         "aggs": {"a": {"avg": {"field": "tenant_id"}}}}}}}
PERCENTILES = {"p": {"percentiles": {"field": "tenant_id", "percents": [10, 50, 99]}}}
COMPOSITE = {"c": {"composite": {"size": 5, "sources": [{"sev": {"terms": {"field": "severity_text"}}},
                                                         {"ten": {"terms": {"field": "tenant_id"}}}],
                                 "after": {"sev": "ERROR", "ten": 17}}}}
SEARCH_AFTER = {"split_id": "", "segment_ord": 0, "doc_id": 0, "sort_value": ("u64", 50)}
# shape -> (query, request fields)
SHAPES = {
    "score_topk": (OR4, dict(max_hits=40, sort_fields=[("_score", proto.DESC)])),
    "column_sort_search_after": (term("t1"), dict(max_hits=30, sort_fields=[("tenant_id", proto.ASC)], search_after=SEARCH_AFTER)),
    "terms_date_histogram_avg": (term("t0"), dict(max_hits=0, aggs=TERMS_HIST_AVG)),
    "percentiles": (term("t1"), dict(max_hits=5, sort_fields=[("timestamp", proto.DESC)], aggs=PERCENTILES)),
    "composite_after": (term("t0"), dict(max_hits=0, aggs=COMPOSITE)),
    "count_only": (term("t2"), dict(max_hits=0)),
    "count_hits_underestimate": (term("t1"), dict(max_hits=10, sort_fields=[("timestamp", proto.ASC)], count_hits=1)),
}


@pytest.fixture(scope="module")
def corpus(gpu_ctx):
    imgs = [S.synth_split(20_000 + 97 * i, 300 + i, FRACS, split_id=f"lc-{i:02d}", ts_start_secs=T0 + DAY * i, ts_span_secs=DAY)
            for i in range(N_SPLITS)]
    for im in imgs:
        gpu_ctx.register_split(im)
    return imgs


@pytest.fixture
def cache_on(gpu_ctx):
    gpu_ctx.set_leaf_cache_budget(BUDGET)
    try:
        yield gpu_ctx
    finally:
        gpu_ctx.set_leaf_cache_budget(0)


def offsets(imgs):
    return [proto.enc_split_offsets(im.split_id, im.num_docs, timestamp_start=T0 + DAY * int(im.split_id[3:]),
                                    timestamp_end=T0 + DAY * (int(im.split_id[3:]) + 1) - 1) for im in imgs]


def leaf_request(imgs, shape, window=None):
    q, kw = SHAPES[shape]
    kw = dict(kw)
    aggs = kw.pop("aggs", None)
    if aggs is not None:
        kw["aggregation_request"] = json.dumps(aggs)
    if window is not None:
        kw.update(start_timestamp=T0 + DAY * window + DAY // 2, end_timestamp=T0 + DAY * (window + 8) + DAY // 2)
    return proto.enc_leaf_search_request(proto.enc_search_request(json.dumps(q), **kw), offsets(imgs), DM)


def view(resp, shape):
    """Everything of a leaf response that the cache must not change."""
    d = proto.dec_leaf_search_response(resp)
    aggs = SHAPES[shape][1].get("aggs")
    fin = None
    if aggs is not None:
        fin = json.loads(service.finalize_aggregation(json.dumps(aggs), d["intermediate_aggregation_result"] or b""))
    return dict(num_hits=d["num_hits"], partial_hits=d["partial_hits"], failed_splits=d["failed_splits"],
                attempted=d["num_attempted_splits"], successful=d["num_successful_splits"], aggs=fin)


def cache_splits(resp):
    rs = proto.dec_leaf_search_response(resp)["resource_stats"] or {}
    return rs.get("partial_result_cache_num_splits", 0)


def looked_up_keys(lreq):
    return {r["key"] for r in service.leaf_cache_keys(lreq) if r["looked_up"]}


@pytest.mark.parametrize("shape", list(SHAPES))
def test_repeat_and_slide(gpu_ctx, corpus, shape):
    r0, r1 = leaf_request(corpus, shape, window=3), leaf_request(corpus, shape, window=4)
    want0, want1 = gpu_ctx.leaf_search(r0), gpu_ctx.leaf_search(r1)  # the cache is off
    assert view(want0, shape)["successful"] > 0
    gpu_ctx.set_leaf_cache_budget(BUDGET)
    try:
        i0 = gpu_ctx.leaf_cache_info()
        first = gpu_ctx.leaf_search(r0)
        i1 = gpu_ctx.leaf_cache_info()
        keys0 = looked_up_keys(r0)
        assert view(first, shape) == view(want0, shape)
        assert cache_splits(first) == 0 and i1["hits"] == i0["hits"] and i1["fills"] - i0["fills"] == len(keys0)
        # the repeat: every split from the cache
        again = gpu_ctx.leaf_search(r0)
        i2 = gpu_ctx.leaf_cache_info()
        assert view(again, shape) == view(want0, shape)
        assert cache_splits(again) == len(keys0) and i2["hits"] - i1["hits"] == len(keys0) and i2["fills"] == i1["fills"]
        rs = proto.dec_leaf_search_response(again)["resource_stats"]
        assert rs.get("localexec_num_splits", 0) == 0 and "split_resources_sum" not in rs  # nothing ran on the device
        # the window slides by one split's span: the splits both windows cover whole hit, the edges miss
        keys1 = looked_up_keys(r1)
        expect_hits = len(keys1 & keys0)
        assert 0 < expect_hits < len(keys1)
        slid = gpu_ctx.leaf_search(r1)
        i3 = gpu_ctx.leaf_cache_info()
        assert view(slid, shape) == view(want1, shape)
        assert cache_splits(slid) == expect_hits and i3["hits"] - i2["hits"] == expect_hits
        assert i3["fills"] - i2["fills"] == len(keys1) - expect_hits
    finally:
        gpu_ctx.set_leaf_cache_budget(0)


def test_invoke_leaf_search_returns_cached_split_results(cache_on, corpus):
    """Seam B: a hit is that split's cached response, with the cache-hit counters as its resource stats."""
    lreq = leaf_request(corpus[:6], "percentiles", window=1)
    cache_on.set_leaf_cache_budget(0)
    want = proto.dec_lambda_responses(cache_on.invoke_leaf_search(lreq))
    cache_on.set_leaf_cache_budget(BUDGET)
    first = proto.dec_lambda_responses(cache_on.invoke_leaf_search(lreq))
    again = proto.dec_lambda_responses(cache_on.invoke_leaf_search(lreq))
    docs = {im.split_id: im.num_docs for im in corpus}
    for w, f, a in zip(want, first, again):
        assert w["split_id"] == f["split_id"] == a["split_id"] and w["error"] is None and a["error"] is None
        for k in ("num_hits", "partial_hits", "intermediate_aggregation_result", "num_attempted_splits", "num_successful_splits"):
            assert w["response"][k] == f["response"][k] == a["response"][k], k
        assert f["response"]["resource_stats"]["localexec_num_splits"] == 1
        assert a["response"]["resource_stats"] == {"partial_result_cache_num_splits": 1, "partial_result_cache_num_docs": docs[a["split_id"]]}


def test_evicted_split_is_served_from_the_cache():
    """Residency eviction keeps the cache's entries: a hit needs no device data. A miss on an evicted split still
    fails, retryably."""
    imgs = [S.synth_split(15_000, 400 + i, FRACS, split_id=f"lc-{i:02d}", ts_start_secs=T0 + DAY * i, ts_span_secs=DAY) for i in range(3)]
    ctx = SearcherContext(0)
    try:
        ctx.set_leaf_cache_budget(BUDGET)
        ctx.register_split(imgs[0])
        ctx.register_split(imgs[1])
        ctx.set_residency_budget(ctx.resident_bytes() + ctx.resident_bytes() // 4)
        lreq = leaf_request(imgs[:2], "terms_date_histogram_avg")
        first = ctx.leaf_search(lreq)
        ctx.register_split(imgs[2])  # evicts the least recently searched split
        gone = [im.split_id for im in imgs[:2] if not ctx.is_resident(im.split_id)]
        assert len(gone) == 1 and ctx.residency_info()["evictions"] == 1
        again = ctx.leaf_search(lreq)
        assert view(again, "terms_date_histogram_avg") == view(first, "terms_date_histogram_avg")
        assert cache_splits(again) == 2
        miss = proto.dec_leaf_search_response(ctx.leaf_search(leaf_request(imgs[:2], "count_only")))
        assert [(f["split_id"], f["retryable_error"]) for f in miss["failed_splits"]] == [(gone[0], True)]
        assert miss["num_successful_splits"] == 1 and miss["num_attempted_splits"] == 2
    finally:
        ctx.close()


def count_request(img, value):
    return proto.enc_leaf_search_request(proto.enc_search_request(json.dumps(term(value))), offsets([img]), DM)


def test_budgets_and_lru(gpu_ctx, corpus):
    img = corpus[0]
    reqs = [count_request(img, f"t{i}") for i in range(4)]
    try:
        # budget 0: no lookup, no entry
        i0 = gpu_ctx.leaf_cache_info()
        gpu_ctx.leaf_search(reqs[0])
        gpu_ctx.leaf_search(reqs[0])
        assert gpu_ctx.leaf_cache_info() == i0 and i0["entries"] == 0 and i0["budget_bytes"] == 0
        # the size of one response
        gpu_ctx.set_leaf_cache_budget(BUDGET)
        gpu_ctx.leaf_search(reqs[0])
        one = gpu_ctx.leaf_cache_info()["used_bytes"]
        assert gpu_ctx.leaf_cache_info()["entries"] == 1 and one > 0
        # below one response: nothing is stored
        gpu_ctx.set_leaf_cache_budget(0)
        gpu_ctx.set_leaf_cache_budget(one - 1)
        f0 = gpu_ctx.leaf_cache_info()["fills"]
        gpu_ctx.leaf_search(reqs[0])
        gpu_ctx.leaf_search(reqs[0])
        info = gpu_ctx.leaf_cache_info()
        assert info["entries"] == 0 and info["fills"] == f0 and info["used_bytes"] == 0
        # room for two responses (every count response of this split has the same size): LRU order
        gpu_ctx.set_leaf_cache_budget(0)
        gpu_ctx.set_leaf_cache_budget(2 * one + one // 2)
        for r in (reqs[0], reqs[1]):
            gpu_ctx.leaf_search(r)
        assert gpu_ctx.leaf_cache_info()["entries"] == 2
        h0 = gpu_ctx.leaf_cache_info()["hits"]
        assert cache_splits(gpu_ctx.leaf_search(reqs[0])) == 1  # t0 is now the most recent
        e0 = gpu_ctx.leaf_cache_info()["evictions"]
        gpu_ctx.leaf_search(reqs[2])  # evicts t1, the least recently used
        info = gpu_ctx.leaf_cache_info()
        assert info["entries"] == 2 and info["evictions"] == e0 + 1 and info["hits"] == h0 + 1
        assert cache_splits(gpu_ctx.leaf_search(reqs[0])) == 1
        assert cache_splits(gpu_ctx.leaf_search(reqs[2])) == 1
        assert cache_splits(gpu_ctx.leaf_search(reqs[1])) == 0
        # registering the split again drops its entries; unregistering does too
        gpu_ctx.set_leaf_cache_budget(BUDGET)
        gpu_ctx.leaf_search(reqs[3])
        assert gpu_ctx.leaf_cache_info()["entries"] >= 1
        gpu_ctx.register_split(img)
        assert gpu_ctx.leaf_cache_info()["entries"] == 0
        assert cache_splits(gpu_ctx.leaf_search(reqs[3])) == 0
        other = S.synth_split(5_000, 499, FRACS, split_id="lc-99", ts_start_secs=T0 + DAY * 99, ts_span_secs=DAY)
        gpu_ctx.register_split(other)
        gpu_ctx.leaf_search(count_request(other, "t0"))
        n = gpu_ctx.leaf_cache_info()["entries"]
        gpu_ctx.unregister_split("lc-99")
        assert gpu_ctx.leaf_cache_info()["entries"] == n - 1
    finally:
        gpu_ctx.set_leaf_cache_budget(0)


def test_concurrent_callers(cache_on, corpus):
    """16 callers at once, mixing hits and misses: every response equals its uncached counterpart."""
    calls = [(shape, w) for shape in SHAPES for w in (2, 3, 4, 9)]
    reqs = {c: leaf_request(corpus, c[0], window=c[1]) for c in calls}
    cache_on.set_leaf_cache_budget(0)
    want = {c: view(cache_on.leaf_search(r), c[0]) for c, r in reqs.items()}
    cache_on.set_leaf_cache_budget(BUDGET)
    for c in calls[::3]:  # some entries before the callers start
        cache_on.leaf_search(reqs[c])
    work = [calls[(i * 7) % len(calls)] for i in range(4 * len(calls))]

    def run(c):
        return c, view(cache_on.leaf_search(reqs[c]), c[0])

    with ThreadPoolExecutor(max_workers=16) as ex:
        got = list(ex.map(run, work))
    for c, v in got:
        assert v == want[c], c
    info = cache_on.leaf_cache_info()
    assert info["hits"] > 0 and info["misses"] > 0


def test_full_hit_launches_no_kernel(corpus):
    """The engine's own launch count (QWGPU_TRACE) for a call that every split answers from the cache: zero."""
    script = textwrap.dedent(f"""
        import json, sys
        sys.path.insert(0, {os.path.dirname(os.path.abspath(__file__))!r})
        import test_gpu_leaf_cache as T
        from quickwit_b200 import splitgen as S
        from quickwit_b200.service import SearcherContext
        imgs = [S.synth_split(10_000, 450 + i, T.FRACS, split_id=f"lc-{{i:02d}}", ts_start_secs=T.T0 + T.DAY * i) for i in range(4)]
        ctx = SearcherContext(0)
        for im in imgs:
            ctx.register_split(im)
        ctx.set_leaf_cache_budget(T.BUDGET)
        r = T.leaf_request(imgs, "terms_date_histogram_avg", window=0)
        ctx.leaf_search(r)
        print("--- second call", file=sys.stderr, flush=True)
        ctx.leaf_search(r)
        ctx.close()
    """)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, QWGPU_TRACE="1", PYTHONPATH=root)
    p = subprocess.run([sys.executable, "-c", script], env=env, cwd=root, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    first, second = p.stderr.split("--- second call")
    line = lambda s: [l for l in s.splitlines() if "leaf_search:" in l][-1]
    assert "4 splits from the cache" not in line(first) and " 0 launches" not in line(first), line(first)
    assert " 0 launches, 4 splits from the cache" in line(second), line(second)
