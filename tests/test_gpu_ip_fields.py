"""`ip` fields on the device. The compiled plans of test_ip_fields_host.py's requests run on the GPU and must equal
the CPU oracle bit for bit (hits, sort values, aggregation cells) on every kernel route they reach: an ip range as
the whole query, as a filter beside a BM25 union, under a term in k_driver, and inside a bool on k_window, selective
and broad; terms on indexed-only fields; terms(ip) alone and nested under date_histogram (hashed cells). Leaf requests
over 64 splits go through qwgpu_leaf_search and the device merge, search_after pages run with the predicate cache
on, and the reference's golden documents run end to end through protobuf, all against the CPU pipeline and the
brute force of ip_ref.py."""
import json
import random

import pytest

from quickwit_b200 import ffi, proto, service, splitgen as S
from quickwit_b200.proto import ASC, DESC
from quickwit_b200.service import SearcherContext
from oracle import oracle as O
from helpers import assert_same
from pipeline import MATCH_ALL, bool_, cpu_split_response, full_text, leafify, search_request, term
import ip_ref as R
import test_ip_fields_host as H

pytestmark = pytest.mark.gpu

DM = H.mapping()
DM_JSON = json.dumps(DM)
ONLY = {"field_mappings": DM["field_mappings"] + [{"name": "peer", "type": "ip"}], "timestamp_field": "ts"}
ONLY_JSON = json.dumps(ONLY)


def big_corpus():
    pool = sorted(H.addresses(300, 41), key=R.v6)
    docs = H.corpus(30_000, 42, pool)
    rnd = random.Random(43)
    for d in docs:  # an indexed-only field beside the fast one
        if rnd.random() < 0.7:
            d["peer"] = rnd.choice(pool[:50])
    return pool, docs


@pytest.fixture(scope="module")
def big(gpu_ctx):
    pool, docs = big_corpus()
    img = S.build_split(docs, ONLY, "ip-gpu-big")
    gpu_ctx.register_split(img)
    yield pool, docs, img
    gpu_ctx.unregister_split(img.split_id)


def device_vs_oracle(ctx, img, ast, dm_json, **kw):
    plan = service.compile_plan(img, search_request(ast, **kw), dm_json)
    got = ctx.split_search([img.split_id], [plan])[0]
    want = O.split_search(img, plan)
    assert_same(got, want, ctx=json.dumps(ast)[:200])
    return got, want


def shapes(pool):
    """pool: addresses in address order"""
    lo, hi = pool[40], pool[200]
    narrow = (pool[100], pool[102])
    rng = H.rng_q("client_ip", lo, hi)
    return {
        "range alone": (rng, [("status", ASC)], 0),
        "narrow range alone": (H.rng_q("client_ip", *narrow), [("_doc", DESC)], 0),
        "ipv4 only": (H.rng_q("client_ip", "0.0.0.0", "255.255.255.255", True, False), [("ts", DESC)], 0),
        "range beside a BM25 union": (bool_(should=[full_text("log", "alpha"), full_text("log", "gamma")], filter=[rng]), [("_score", DESC)], 0),
        "range under a term": (bool_(must=[term("log", "beta")], filter=[rng]), [("_doc", DESC)], QWGPU_KERNEL_DRIVER),
        "ip term under a term": (bool_(must=[term("log", "beta")], filter=[term("client_ip", pool[120])]), [("ts", ASC)], QWGPU_KERNEL_DRIVER),
        "bool on k_window": (bool_(should=[term("client_ip", pool[7]), H.rng_q("client_ip", *narrow), term("log", "gamma")],
                                   must_not=[H.rng_q("client_ip", "10.0.0.0", "10.255.255.255")], minimum_should_match=1), [("status", DESC)], 0),
        "narrow bool on k_window": (bool_(must=[H.rng_q("client_ip", *narrow)], must_not=[term("log", "gamma")],
                                          should=[H.exists_q("client_ip")]), [("_doc", ASC)], 0),
        "exists": (H.exists_q("client_ip"), [("_doc", DESC)], 0),
        "term set": (H.term_set_q("client_ip", pool[10:60:7]), [("_doc", DESC)], 0),
        "indexed-only term": (term("peer", pool[3]), [("_doc", DESC)], 0),
        "indexed-only term beside a BM25 clause": (bool_(must=[full_text("log", "alpha")], filter=[full_text("peer", pool[4])]), [("_score", DESC)], 0),
    }


QWGPU_KERNEL_DRIVER = 2
QWGPU_KERNEL_HASHED_AGGS = 256


@pytest.mark.parametrize("name", list(shapes(sorted(H.addresses(300, 41), key=R.v6)).keys()))
def test_queries_match_oracle_and_brute_force(gpu_ctx, big, name):
    pool, docs, img = big
    ast, sort, route = shapes(pool)[name]
    for K in (10, 1000):
        got, _ = device_vs_oracle(gpu_ctx, img, ast, ONLY_JSON, max_hits=K, sort_fields=sort)
        if route:
            assert got.kernel_mask & route, (name, got.kernel_mask)
    if name == "range alone":
        want = R.range_docs(docs, "client_ip", pool[40], pool[200])
        assert got.num_hits == len(want) > 1000
    if name == "indexed-only term":
        assert got.num_hits == len(R.term_docs(docs, "peer", pool[3])) > 0


@pytest.mark.parametrize("aggs", [
    {"ips": {"terms": {"field": "client_ip", "size": 10}}},
    {"ips": {"terms": {"field": "client_ip", "size": 20, "order": {"_key": "desc"}, "missing": "::1"}}},
    {"ips": {"terms": {"field": "client_ip"}, "aggs": {"s": {"stats": {"field": "status"}}}}},
], ids=["terms", "terms-key-missing", "terms-stats"])
def test_terms_cells_match_oracle(gpu_ctx, big, aggs):
    pool, docs, img = big
    for ast in (MATCH_ALL, H.rng_q("client_ip", pool[10], pool[250])):
        device_vs_oracle(gpu_ctx, img, ast, ONLY_JSON, max_hits=0, aggs=aggs)


def leaf(ctx, imgs, ast, dm_json, **kw):
    sreq = search_request(ast, **leafify(kw))
    lreq = proto.enc_leaf_search_request(sreq, [proto.enc_split_offsets(im.split_id, im.num_docs) for im in imgs], dm_json)
    return sreq, ctx.leaf_search(lreq)


def cpu_leaf(imgs, sreq, dm):
    return service.merge_leaf_responses(sreq, [cpu_split_response(im, sreq, dm) for im in imgs])


def finalize(aggs, resp):
    inter = proto.dec_leaf_search_response(resp)["intermediate_aggregation_result"]
    return json.loads(service.finalize_aggregation(json.dumps(aggs), inter or b""))


def test_nested_terms_hashed(gpu_ctx, big):
    """terms(ip) below two bucket levels: the plan takes the hashed cells, whose entries carry raw ordinals"""
    pool, docs, img = big
    ips = {"terms": {"field": "client_ip", "size": 5, "split_size": 100000, "order": {"_key": "asc"}}}
    aggs = {"t": {"date_histogram": {"field": "ts", "fixed_interval": "3h"},
                  "aggs": {"st": {"terms": {"field": "status"}, "aggs": {"ips": ips}}}}}
    plan = service.compile_plan(img, search_request(MATCH_ALL, max_hits=0, aggs=aggs), ONLY_JSON)
    r = gpu_ctx.split_search([img.split_id], [plan])[0]
    assert r.kernel_mask & QWGPU_KERNEL_HASHED_AGGS
    sreq, resp = leaf(gpu_ctx, [img], MATCH_ALL, ONLY_JSON, max_hits=0, aggs=aggs)
    got = finalize(aggs, resp)
    assert got == finalize(aggs, cpu_leaf([img], sreq, ONLY))
    n = 0
    for b in got["t"]["buckets"]:
        lo = b["key"] / 1000
        for sb in b["st"]["buckets"]:
            matched = [(docs, [d for d in range(len(docs)) if lo <= docs[d]["ts"] < lo + 3 * 3600 and docs[d]["status"] == sb["key"]])]
            assert sb["ips"] == R.terms_result(R.terms_counts(matched, "client_ip"), 5, "_key", False)
            n += 1
    assert n > 20


@pytest.fixture(scope="module")
def many(gpu_ctx):
    splits = H.split_set(64, 51)
    imgs = [img for _, img in splits]
    for im in imgs:
        gpu_ctx.register_split(im)
    yield splits
    for im in imgs:
        gpu_ctx.unregister_split(im.split_id)


@pytest.mark.parametrize("sort", [[("_doc", DESC)], [("status", ASC), ("ts", DESC)], [("_score", DESC)]], ids=["doc", "status+ts", "score"])
def test_64_splits_leaf_search(gpu_ctx, many, sort):
    imgs = [img for _, img in many]
    pool = sorted({a for docs, _ in many for doc in docs for a in R.values(doc, "client_ip")})
    lo, hi = str(pool[len(pool) // 5]), str(pool[4 * len(pool) // 5])
    aggs = {"ips": {"terms": {"field": "client_ip", "size": 25, "split_size": 100000}}}
    ast = bool_(must=[full_text("log", "alpha")], filter=[H.rng_q("client_ip", lo, hi)])
    sreq, resp = leaf(gpu_ctx, imgs, ast, DM_JSON, max_hits=50, sort_fields=sort, aggs=aggs)
    got, want = proto.dec_leaf_search_response(resp), proto.dec_leaf_search_response(cpu_leaf(imgs, sreq, DM))
    assert got["num_hits"] == want["num_hits"] and got["partial_hits"] == want["partial_hits"]
    assert finalize(aggs, resp) == finalize(aggs, cpu_leaf(imgs, sreq, DM))
    matched = [(docs, [d for d in R.range_docs(docs, "client_ip", lo, hi) if "alpha" in docs[d]["log"].split()]) for docs, _ in many]
    assert got["num_hits"] == sum(len(m) for _, m in matched)
    assert finalize(aggs, resp)["ips"] == R.terms_result(R.terms_counts(matched, "client_ip"), 25)


def test_search_after_pages_with_predicate_cache(many):
    imgs = [img for _, img in many][:8]
    on = SearcherContext(0)
    try:
        on.set_predicate_cache_budget(1 << 28)
        for im in imgs:
            on.register_split(im)
        pool = sorted({a for docs, _ in many[:8] for doc in docs for a in R.values(doc, "client_ip")})
        ast = bool_(must=[H.rng_q("client_ip", str(pool[3]), str(pool[-3]))], must_not=[term("client_ip", str(pool[10]))])
        kw = dict(max_hits=37, sort_fields=[("ts", DESC)])
        sa, seen, fills = None, [], 0
        while True:
            args = dict(kw, search_after=sa) if sa else kw
            sreq, resp = leaf(on, imgs, ast, DM_JSON, **args)
            got = proto.dec_leaf_search_response(resp)
            want = proto.dec_leaf_search_response(cpu_leaf(imgs, sreq, DM))
            assert got["num_hits"] == want["num_hits"] and got["partial_hits"] == want["partial_hits"]
            if not got["partial_hits"]:
                break
            seen += got["partial_hits"]
            sa = got["partial_hits"][-1]
        info = on.predicate_cache_info()
        assert info["fills"] > 0 and info["hits"] > 0, info
        total = sum(len(R.range_docs(docs, "client_ip", str(pool[3]), str(pool[-3])))
                    - len(set(R.range_docs(docs, "client_ip", str(pool[3]), str(pool[-3]))) & set(R.term_docs(docs, "client_ip", str(pool[10]))))
                    for docs, _ in many[:8])
        assert len(seen) == total
    finally:
        on.close()


def test_golden_documents_end_to_end(gpu_ctx):
    for dm, name in ((H.GOLDEN_INDEXED, "golden-indexed"), (H.GOLDEN_FAST, "golden-fast")):
        img = S.build_split(H.GOLDEN_DOCS, dm, name)
        gpu_ctx.register_split(img)
        try:
            dj = json.dumps(dm)
            for ast, want in ((MATCH_ALL, [0, 1, 2, 3, 4, 5]), (full_text("host", "10.10.11.125"), [2]),
                              (H.rng_q("host", "10.0.0.0", "10.255.255.255"), [1, 2, 5])):
                if dm is H.GOLDEN_INDEXED and ast.get("type") == "range":
                    continue
                _, resp = leaf(gpu_ctx, [img], ast, dj, max_hits=10)
                r = proto.dec_leaf_search_response(resp)
                assert r["num_hits"] == len(want) and sorted(h["doc_id"] for h in r["partial_hits"]) == want, (name, ast)
            if dm is H.GOLDEN_FAST:
                aggs = {"hosts": {"terms": {"field": "host", "order": {"_key": "asc"}}}}
                _, resp = leaf(gpu_ctx, [img], MATCH_ALL, dj, max_hits=0, aggs=aggs)
                assert finalize(aggs, resp)["hosts"]["buckets"] == [
                    {"doc_count": 1, "key": "::afff:4567:890a"}, {"doc_count": 1, "key": "10.10.11.125"},
                    {"doc_count": 2, "key": "10.10.12.123"}, {"doc_count": 1, "key": "192.168.0.1"},
                    {"doc_count": 1, "key": "2001:db8::1:0:0:1"}]
        finally:
            gpu_ctx.unregister_split(img.split_id)
