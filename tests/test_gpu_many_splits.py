"""Leaf requests over hundreds of splits on the GPU, against a brute force over every document of every split.

A searcher receives one leaf request for every split the root assigns to it, often hundreds. The engine runs them in
one launch sequence and merges the per-split top-K lists on the device (k_merge_prep / k_merge). Code there only runs
at high list counts: k_merge's lanes take a second round of lists from 33 lists on, k_merge_prep stops pruning above
64 lists, and k_union finds a work item's split in 32-split ballots. Base images are registered under many split ids
(many_splits_ref): twins tie on every sort value, so only the (split id, doc id) tie-break orders them, and the ids'
lexical order differs from the request order and from the registration order.

- the device merge through qwgpu_leaf_search, at 1 to 300 lists and K from 1 to 20 000, for every sort kind and list
  shape, against many_splits_ref.expected and the CPU pipeline;
- every kernel route with 65 to 300 splits in one seam-C call, each split bit-identical to the oracle;
- per-split fates (failed, evicted, empty, NONE, pruned, demoted, counted from metadata) mixed in one leaf request;
- aggregations over 100 splits against counts computed from the documents."""
import json

import numpy as np
import pytest

from quickwit_b200 import ffi, plan as P, proto, service, splitgen as S
from quickwit_b200.proto import ASC, DESC
from oracle import oracle as O
from helpers import assert_same
from pipeline import MATCH_ALL, bool_, cpu_root_search, cpu_split_response, search_request, term
from regex_ref import oracle_search
import many_splits_ref as R

pytestmark = pytest.mark.gpu

NS = (1, 2, 31, 32, 33, 63, 64, 65, 96, 129, 300)
BIG_DOCS = 1 << 20


def ks(n):
    """max_hits + start_offset of every merge case at n lists."""
    return sorted({1, n - 1, n, n + 1, 100, 4096, 4097, 20_000} - {0})


class Corpus:
    """The base images, and the split ids registered on the context (each under exactly one base)."""

    def __init__(self, ctx):
        self.ctx = ctx
        self.hand = {n: R.Base(R.hand_split(n, i, f"hand-{n}", with_c=n != 15_360)) for i, n in enumerate(R.HAND_DOCS)}
        self.h40b = R.Base(R.hand_split(40_000, 11, "hand-40k-b", with_c=False))
        self.solo = R.Base(R.hand_split(40_000, 12, "hand-solo", solo=True))
        self.big = R.Base(R.hand_split(BIG_DOCS, 13, "hand-big"))
        self.synth = [R.Base(R.synth(i, 3000 + 97 * i)) for i in range(70)]
        self.registered = {}

    def pool(self):
        """The mixed shape's bases, in the order request positions take them."""
        h = self.hand
        return [h[40_000], h[127], self.big, h[15_359], h[15_360], self.h40b, h[15_361], h[1], h[0]] + self.synth

    def register(self, entries):
        """Registers the entries' ids that are not yet registered, in an order unrelated to the request's."""
        todo = [(sid, b) for sid, b in entries if sid not in self.registered]
        for sid, b in entries:
            assert self.registered.get(sid, b) is b, sid
        for k in np.random.default_rng(len(self.registered)).permutation(len(todo)):
            sid, b = todo[k]
            self.ctx.register_split(b.img, split_id=sid)
            self.registered[sid] = b
        return entries

    def mixed(self, n):
        pool = self.pool()
        return self.register([(sid, pool[i % len(pool)]) for i, sid in R.ids("m", n, 1)])

    def twins(self, n, base=None, prefix="w"):
        return self.register([(sid, base or self.hand[40_000]) for _, sid in R.ids(prefix, n, 2)])

    def single(self, n):
        """One split holds the `solo` term; the rest are twins without it."""
        e = [(sid, self.hand[40_000]) for _, sid in R.ids("w", n, 2)]
        e[n // 2] = ("solo-0", self.solo)
        return self.register(e)

    def timed(self, n):
        """The 70 time-partitioned synthetic splits, then twins of the 40k hand-made split (day 0)."""
        e = [(f"t-{i}", b) for i, b in enumerate(self.synth[:n])] + [(sid, self.hand[40_000]) for _, sid in R.ids("w", max(0, n - 70), 2)]
        order = np.random.default_rng(3).permutation(len(e))
        return self.register([e[i] for i in order])

    def close(self):
        for sid in self.registered:
            self.ctx.unregister_split(sid)


@pytest.fixture(scope="module")
def corpus(gpu_ctx):
    gpu_ctx.set_max_hits(20_000)
    c = Corpus(gpu_ctx)
    yield c
    c.close()
    gpu_ctx.set_max_hits(4096)


def leaf(ctx, entries, ast, sort, K, start=0, **kw):
    """One qwgpu_leaf_search over `entries`, merged to the root's page: (decoded root response, decoded leaf response)."""
    lreq, root = R.leaf_request(entries, ast, sort, K - start, start, **kw)
    resp = ctx.leaf_search(lreq)
    return proto.dec_leaf_search_response(service.merge_leaf_responses(root, [resp])), proto.dec_leaf_search_response(resp)


def check(ctx, entries, ast, sort, K, start, tag, cross=True, **kw):
    got, lf = leaf(ctx, entries, ast, sort, K, start, **kw)
    nh, want = R.expected(entries, ast, sort, K)
    assert lf["num_successful_splits"] == len(entries) and not lf["failed_splits"], tag
    # the leaf response carries the device merge's own order (the root merge below sorts its hits again)
    assert lf["num_hits"] == nh and R.hits_of(lf) == want, f"{tag}: the leaf response differs from the brute force"
    assert got["num_hits"] == nh, f"{tag}: num_hits {got['num_hits']} != {nh}"
    g = R.hits_of(got)
    if g != want[start:]:
        bad = next((i for i, (a, b) in enumerate(zip(g, want[start:])) if a != b), min(len(g), len(want) - start))
        raise AssertionError(f"{tag}: {len(g)} hits against {len(want) - start}; first difference at {bad}: "
                             f"{g[bad] if bad < len(g) else None} != {want[start + bad] if start + bad < len(want) else None}")
    if cross:
        imgs = [S.SplitImage(b.img.array, sid) for sid, b in entries]
        w = cpu_root_search(imgs, ast, R.MAPPING, max_hits=K - start, start_offset=start, sort_fields=list(sort), **kw)
        assert w["num_hits"] == got["num_hits"] and w["partial_hits"] == got["partial_hits"], f"{tag}: differs from the CPU pipeline"
    return got


def cheap(n, K):
    """Whether the CPU pipeline's cross-check stays within a second or so."""
    return n * min(K, 4096) <= 150_000


# ---- 1. the device merge through qwgpu_leaf_search ----------------------------------------------------------------------
@pytest.mark.parametrize("n", NS)
def test_merge_list_counts(corpus, n):
    """Mixed bases (0 to 1 M docs, some without column c) at every K, with and without a start offset."""
    e = corpus.mixed(n)
    for j, K in enumerate(ks(n)):
        start = K // 3 if j % 2 else 0
        check(corpus.ctx, e, term("body", "t0"), [("c", DESC)], K, start, f"n={n} K={K} start={start}", cross=cheap(n, K))


SORTS = {"score_desc": [("_score", DESC)], "score_asc": [("_score", ASC)], "doc_asc": [("_doc", ASC)],
         "doc_desc": [("_doc", DESC)], "c_desc": [("c", DESC)], "c_asc": [("c", ASC)],
         "two_keys": [("tenant_id", ASC), ("c", DESC)], "two_keys_c_first": [("c", DESC), ("tenant_id", ASC)]}


@pytest.mark.parametrize("sort", list(SORTS))
@pytest.mark.parametrize("shape", ["twins", "mixed"])
def test_merge_sorts(corpus, sort, shape):
    """Every sort kind. Twins tie on every value, including f32 scores; the mixed shape has lists of None values."""
    for n in (33, 65, 129, 300):
        e = corpus.twins(n) if shape == "twins" else corpus.mixed(n)
        for K, start in ((n, 0), (4097, 97), (100, 0) if n < 300 else (20_000, 5)):
            check(corpus.ctx, e, term("body", "t1"), SORTS[sort], K, start, f"{shape} {sort} n={n} K={K} start={start}", cross=cheap(n, K))


@pytest.mark.parametrize("order", [DESC, ASC])
def test_merge_time_partitioned(corpus, order):
    """70 splits with disjoint time ranges (plus twins at day 0): the whole top K of a descending sort comes from the
    last split, which holds K hits by itself; ascending, from the ties of the twins."""
    for n in (65, 70, 129):
        e = corpus.timed(n)
        for K, start in ((1, 0), (n, 0), (500, 10), (4097, 0), (20_000, 100)):
            got = check(corpus.ctx, e, term("body", "t0"), [("timestamp", order)], K, start, f"time n={n} K={K}", cross=cheap(n, K))
            if order == DESC and K <= 500:
                assert {h["split_id"] for h in got["partial_hits"]} == {f"t-{min(n, 70) - 1}"}


@pytest.mark.parametrize("n", (33, 65, 129, 300))
def test_merge_list_shapes(corpus, n):
    """One non-empty list among n; lists shorter than ceil(K / non-empty) (10 hits each); every list empty."""
    for K in (1, 100, 4097):
        check(corpus.ctx, corpus.single(n), term("body", "solo"), [("c", DESC)], K, 0, f"single n={n} K={K}", cross=cheap(n, K))
        check(corpus.ctx, corpus.twins(n), term("body", "t2"), [("c", ASC)], K, 0, f"short n={n} K={K}", cross=cheap(n, K))
        check(corpus.ctx, corpus.twins(n), term("body", "t2"), [("_score", DESC)], K, 0, f"short score n={n} K={K}", cross=cheap(n, K))
        got = check(corpus.ctx, corpus.mixed(n), term("body", "absent"), [("c", DESC)], K, 0, f"empty n={n} K={K}", cross=False)
        assert got["num_hits"] == 0 and got["partial_hits"] == []


# ---- 2. every route with 65 to 300 splits in one seam-C call -------------------------------------------------------------
_ORACLE = {}


def seam_c(ctx, entries, make_plan, kernel, tag, oracle=O.split_search):
    """One split_search over every entry; each split's result equals the oracle's (computed once per base and plan)."""
    plans = [make_plan(sid, b) for sid, b in entries]
    res = ctx.split_search([sid for sid, _ in entries], plans)
    for (sid, b), pl, r in zip(entries, plans, res):
        key = (id(b), pl)
        if key not in _ORACLE:
            _ORACLE[key] = oracle(b.img, pl)
        assert_same(r, _ORACLE[key], ctx=f"{tag} {sid}")
    for (sid, _), r in zip(entries, res):
        if r.num_hits:   # (a split with no match may be answered without a kernel)
            assert r.kernel_mask & kernel, f"{tag} {sid}: kernel_mask={r.kernel_mask:#x}"
    return res[0]


def compiled(ast, **kw):
    req = search_request(ast, **kw)
    return lambda sid, b: service.compile_plan(b.img, req, R.DM, sid)


def _grid():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 2


def test_union_fused_sample(corpus):
    """70 twins of a 1 M-doc split: enough windows for the sample inside k_union's collect pass (two launches)."""
    e = corpus.twins(70, corpus.big, "b")
    ast = bool_(should=[term("body", "t0"), term("body", "t1")])
    for K in (10, 1000):
        r = seam_c(corpus.ctx, e, compiled(ast, max_hits=K, sort_fields=[("_score", DESC)]), ffi.KERNEL_UNION, f"fused K={K}")
        total = 70 * ((BIG_DOCS + 15_359) // 15_360)
        assert total >= 4 * _grid() and r.sample_stride == total // _grid(), r.sample_stride
        assert r.num_kernel_launches == 2 or r.exact_fallbacks == 1, r.num_kernel_launches


W_UNION = 15_360   # docs per k_union window (and per sampled window: W rounded down to 1024)


def test_union_sampled_pass_with_small_splits(corpus):
    """The 1 M-doc split, then 65 twins of the 15 359-doc split, by `_score`: too few windows for the fused sample, so
    k_union runs its separate sampled pass. Its stride comes from the large split (69 windows: 69 // 8 = 8), and split i
    samples the windows w with w % 8 == i % 8, without edge windows: 57 of the one-window twins get no sampled window.
    The large split's BM25 scores take only 154 distinct values, so it takes the exact repair once when searched
    alone, and the batch takes it once too. Every split must equal the oracle."""
    e = [("u-big", corpus.big)] + corpus.twins(65, corpus.hand[15_359], "u")
    corpus.register(e[:1])
    mw = -(-BIG_DOCS // W_UNION)
    stride = max(min(16, mw // 8), min(-(-(mw + 65) // _grid()), 32, mw // 8))
    assert stride == 8 and mw + 65 < 4 * _grid()
    assert sum(1 for i in range(1, len(e)) if i % stride) == 57
    ast = bool_(should=[term("body", "t0"), term("body", "t1")])
    for K in (10, 100):
        plan = compiled(ast, max_hits=K, sort_fields=[("_score", DESC)])
        alone = seam_c(corpus.ctx, e[:1], plan, ffi.KERNEL_UNION, f"union sampled alone K={K}")
        assert alone.sample_stride == stride and alone.exact_fallbacks == 1, (alone.sample_stride, alone.exact_fallbacks)
        r = seam_c(corpus.ctx, e, plan, ffi.KERNEL_UNION, f"union sampled K={K}")
        path = (r.sample_stride, r.num_kernel_launches, r.exact_fallbacks, hex(r.kernel_mask))
        assert r.sample_stride == stride and r.num_kernel_launches > 2 and r.exact_fallbacks == 1, path


def test_window_edge_sample_with_small_splits(corpus):
    """A 1 M-doc split among 299 small ones of every shape (some without column c, some of 0 or 1 docs), served by
    k_window. Its sampled pass takes every stride-th window of each split plus the split's first and last window, so
    every non-empty split is sampled however short it is."""
    e = corpus.mixed(300)
    ast = bool_(should=[term("body", "t0"), term("body", "t1")])
    for K in (10, 1000):
        r = seam_c(corpus.ctx, e, compiled(ast, max_hits=K, sort_fields=[("_score", DESC)]), ffi.KERNEL_WINDOW, f"sampled K={K}")
        assert r.sample_stride >= 2 and r.num_kernel_launches > 2 and r.exact_fallbacks <= 1, (r.sample_stride, r.num_kernel_launches)


ROUTES = {
    "driver": (bool_(must=[term("body", "t1")], filter=[{"type": "range", "field": "tenant_id", "lower_bound": {"Included": 2},
                                                          "upper_bound": {"Included": 9}}]),
               dict(max_hits=200, sort_fields=[("c", DESC)]), ffi.KERNEL_DRIVER),
    "window_must_not": (bool_(must=[term("body", "t0")], must_not=[term("body", "t1")]), dict(max_hits=300, sort_fields=[("c", ASC)]),
                        ffi.KERNEL_WINDOW),
    "window_msm": (bool_(should=[term("body", "t0"), term("body", "t1"), term("body", "t2")], minimum_should_match=2),
                   dict(max_hits=100, sort_fields=[("tenant_id", DESC), ("c", ASC)]), ffi.KERNEL_WINDOW),
    "driver_search_after": (term("body", "t0"), dict(max_hits=100, sort_fields=[("c", DESC)],
                                                     search_after={"split_id": "m-40", "doc_id": 500, "sort_value": ("u64", 30)}),
                            ffi.KERNEL_DRIVER),
    "fast_aggs": (MATCH_ALL, dict(max_hits=0, aggs={"sev": {"terms": {"field": "severity_text"}}, "t": {"stats": {"field": "tenant_id"}},
                                                 "days": {"date_histogram": {"field": "timestamp", "fixed_interval": "1d"}}}),
                ffi.KERNEL_FAST_AGGS),
}


@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("n", (65, 300))
def test_routes(corpus, route, n):
    ast, kw, kernel = ROUTES[route]
    seam_c(corpus.ctx, corpus.mixed(n), compiled(ast, **kw), kernel, f"{route} n={n}")


def test_hashed_aggs_route(corpus):
    """Three nested levels (terms > terms > date_histogram) take the hashed cells on every split of 129: each split's
    aggregation result equals its CPU leaf response."""
    aggs = {"sev": {"terms": {"field": "severity_text"}, "aggs": {"ten": {"terms": {"field": "tenant_id", "size": 20},
                                                                         "aggs": {"d": {"date_histogram": {"field": "timestamp", "fixed_interval": "1d"}}}}}}}
    e = corpus.mixed(129)
    req = search_request(MATCH_ALL, max_hits=0, aggs=aggs)
    plans = [service.compile_plan(b.img, req, R.DM, sid) for sid, b in e]
    res = corpus.ctx.split_search([sid for sid, _ in e], plans)
    for (sid, b), r in zip(e, res):
        assert not b.n or r.kernel_mask & ffi.KERNEL_HASHED_AGGS, f"{sid}: kernel_mask={r.kernel_mask:#x}"
        img = S.SplitImage(b.img.array, sid)
        built = (service.build_leaf_response_entries(img, req, R.DM, r.num_hits, r.hits, r.entries) if r.num_entries
                 else service.build_leaf_response(img, req, R.DM, r.num_hits, r.hits, r.cells))
        got = proto.dec_leaf_search_response(built)
        want = proto.dec_leaf_search_response(cpu_split_response(img, req, R.MAPPING))
        assert got["num_hits"] == want["num_hits"] and got["intermediate_aggregation_result"] == want["intermediate_aggregation_result"], sid


@pytest.fixture(scope="module")
def msg_splits(corpus):
    bases = [R.Base(S.synth_split(20_000 + 1000 * i, 500 + i, R.SYNTH_FRACS, msg_vocab=32, split_id=f"msg-{i}")) for i in range(3)]
    return corpus.register([(sid, bases[i % 3]) for i, sid in R.ids("p", 96, 4)])


def test_phrase_route(corpus, msg_splits):
    ast = {"type": "full_text", "field": "msg", "text": "w0 w1", "params": {"mode": {"type": "phrase", "slop": 0}}, "lenient": False}
    for kw in (dict(max_hits=100, sort_fields=[("_score", DESC)]), dict(max_hits=50, sort_fields=[("timestamp", ASC)])):
        seam_c(corpus.ctx, msg_splits, compiled(ast, **kw), ffi.KERNEL_PHRASE, f"phrase {kw['sort_fields']}")


def test_term_set_route(corpus, msg_splits):
    def make(sid, b):
        ords = sorted(b.img.term_ord("msg", f"w{k}") for k in (3, 5, 8, 13))
        return P.make_plan(P.bool_([P.term_set(b.img, "msg", ords)]), 1000)
    seam_c(corpus.ctx, msg_splits, make, ffi.KERNEL_TERM_SET, "term set", oracle=oracle_search)


# ---- 3. per-split fates in one leaf request ----------------------------------------------------------------------------
def test_split_fates():
    """On a context of its own: a split that is not registered, one evicted by the residency budget, an empty one,
    splits where the query compiles to NONE, splits outside the time range, and splits with hits, in one request of
    120 splits; then the same splits under CountHits::Underestimate demotion and metadata-count answers."""
    ctx = service.SearcherContext(0)
    try:
        h40 = R.Base(R.hand_split(40_000, 21, "f-h40"))
        h127 = R.Base(R.hand_split(127, 22, "f-h127"))
        h0 = R.Base(R.hand_split(0, 23, "f-h0"))
        syn = [R.Base(R.synth(i, 2000 + 13 * i)) for i in range(40)]
        live = [("evicted-0", h40)]   # registered first: the least recently used
        live += [(f"f-syn-{i}", b) for i, b in enumerate(syn)] + [(sid, h127) for _, sid in R.ids("f127", 40, 5)]
        live += [(sid, h40) for _, sid in R.ids("f40", 36, 6)] + [("f-empty", h0)]
        for sid, b in live:
            ctx.register_split(b.img, split_id=sid)
        ctx.set_residency_budget(ctx.resident_bytes())
        ctx.register_split(h40.img, split_id="f-last")         # needs room: evicts evicted-0
        assert not ctx.is_resident("evicted-0") and ctx.residency_info()["evictions"] == 1
        live = [x for x in live if x[0] != "evicted-0"] + [("f-last", h40)]
        ghosts = [("ghost-1", h40), ("evicted-0", h40)]
        entries = live + ghosts
        order = np.random.default_rng(7).permutation(len(entries))
        entries = [entries[i] for i in order]
        assert len(entries) >= 120

        def offsets(kind):
            out = []
            for sid, b in entries:
                v, has = b.column("timestamp")
                secs = (v ^ np.uint64(1 << 63)).astype(np.int64) // 10**9
                lo, hi = (int(secs.min()), int(secs.max())) if b.n else (R.T0, R.T0)
                out.append(proto.enc_split_offsets(sid, b.n, lo, hi) if kind else proto.enc_split_offsets(sid, b.n))
            return out

        # t3 exists only in the synthetic splits: it compiles to NONE on the hand-made ones; the time range keeps days 5..24
        tr = (R.T0 + 6 * R.DAY, R.T0 + 25 * R.DAY)
        for sort, K in (([("timestamp", DESC)], 300), ([("_score", DESC)], 1000), ([("c", ASC)], 50)):
            ast = term("body", "t3")
            lreq = proto.enc_leaf_search_request(search_request(ast, max_hits=K, sort_fields=sort, start_timestamp=tr[0], end_timestamp=tr[1]),
                                                 offsets(True), R.DM)
            resp = proto.dec_leaf_search_response(ctx.leaf_search(lreq))
            failed = sorted((f["split_id"], f["retryable_error"]) for f in resp["failed_splits"])
            assert failed == [("evicted-0", True), ("ghost-1", True)], failed
            assert resp["num_attempted_splits"] == len(entries) and resp["num_successful_splits"] == len(live)
            if sort[0][0] == "_score":
                # the score of the oracle's full hit list knows no time range: check against the CPU pipeline
                imgs = [S.SplitImage(b.img.array, sid) for sid, b in live]
                want = cpu_root_search(imgs, ast, R.MAPPING, max_hits=K, sort_fields=sort, start_timestamp=tr[0], end_timestamp=tr[1])
                assert resp["num_hits"] == want["num_hits"] and resp["partial_hits"] == want["partial_hits"]
                continue
            nh, want = R.expected(live, ast, sort, K, time_range=tr)
            assert resp["num_hits"] == nh and R.hits_of(resp) == want, sort
            names = dict(live)
            for h in resp["partial_hits"]:
                assert h["split_id"] in names and h["doc_id"] < names[h["split_id"]].n
        # match_all by timestamp with CountHits::Underestimate: splits that cannot reach the top are not searched
        lreq = proto.enc_leaf_search_request(search_request(MATCH_ALL, max_hits=20, sort_fields=[("timestamp", DESC)], count_hits=1),
                                             offsets(True), R.DM)
        plan = service.optimize_leaf_request(lreq)
        resp = proto.dec_leaf_search_response(ctx.leaf_search(lreq))
        skipped = {p["split_id"] for p in plan if p["skipped"]}
        assert len(skipped) >= 100, len(skipped)
        searched = [x for x in live if x[0] not in skipped]
        nh, want = R.expected(searched, MATCH_ALL, [("timestamp", DESC)], 20)
        assert R.hits_of(resp) == want and resp["num_hits"] == nh
        assert R.expected(live, MATCH_ALL, [("timestamp", DESC)], 20)[1] == want
        # match_all without hits: every split, resident or not, is counted from its metadata
        lreq = proto.enc_leaf_search_request(search_request(MATCH_ALL, max_hits=0), offsets(False), R.DM)
        resp = proto.dec_leaf_search_response(ctx.leaf_search(lreq))
        assert resp["num_hits"] == sum(b.n for _, b in entries) and not resp["failed_splits"]
        assert resp["num_successful_splits"] == len(entries)
    finally:
        ctx.close()


# ---- 4. aggregations over 100 splits -------------------------------------------------------------------------------------
def test_aggregations(corpus):
    """Terms, date_histogram and stats, and a three-level aggregation on hashed cells, over 129 mixed splits: the
    finalized JSON equals the CPU pipeline's, and its counts equal those computed from the documents."""
    e = corpus.mixed(129)
    aggs = {"sev": {"terms": {"field": "severity_text"}, "aggs": {"ten": {"terms": {"field": "tenant_id", "size": 200},
                                                                         "aggs": {"d": {"date_histogram": {"field": "timestamp", "fixed_interval": "1d"}}}}}},
            "days": {"date_histogram": {"field": "timestamp", "fixed_interval": "1d"}},
            "ten": {"stats": {"field": "tenant_id"}}}
    lreq = proto.enc_leaf_search_request(search_request(MATCH_ALL, max_hits=0, aggs=aggs),
                                         [proto.enc_split_offsets(sid, b.n) for sid, b in e], R.DM)
    root = search_request(MATCH_ALL, max_hits=0, aggs=aggs)
    got = proto.dec_leaf_search_response(service.merge_leaf_responses(root, [corpus.ctx.leaf_search(lreq)]))
    a = json.loads(service.finalize_aggregation(json.dumps(aggs), got["intermediate_aggregation_result"]))
    imgs = [S.SplitImage(b.img.array, sid) for sid, b in e]
    assert a == cpu_root_search(imgs, MATCH_ALL, R.MAPPING, max_hits=0, aggs=aggs)["aggregations"]
    R.check_aggs(a, [b for _, b in e])
