"""Top-K requests of more than 4096 hits (max_hits + start_offset up to 20 000) on the deep selection path
(deep_select_kernel.cuh, DESIGN.md §4.6).

A split that asks for K > 4096 hits keeps qw_cand_cap(K) = 2K (rounded up to 1024) candidates and is finished by the cut /
tile sort / rank kernels instead of k_select. Every result is checked bit for bit against the oracle AND against a
brute force over the arrays the corpus was generated from (numpy lexsort for column sorts, the numpy float32 BM25
restatement for `_score` sorts); the path is asserted from the result's kernel_mask (QWGPU_KERNEL_DEEP_SELECT) and,
on ~1 M-doc splits, from sample_stride / exact_fallbacks / refined / radix_passes. A context serves K up to 4096 until
qwgpu_set_max_hits raises its limit: this module raises it to 20 000 and restores the default when it is done."""
import ctypes as C
import json

import numpy as np
import pytest

from quickwit_b200 import ffi, plan as P, proto, service, splitgen as S
from oracle import oracle as O
from helpers import SCORE_DESC, assert_same, bm25_contributions, bm25_norm, bm25_weight, col_sort
from pipeline import bool_, cpu_root_search, leafify, search_request, term

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _deep_limit(gpu_ctx):
    gpu_ctx.set_max_hits(20_000)
    yield
    gpu_ctx.set_max_hits(4096)

N_SMALL = 200_000      # docs of a route split: more than 20 000 matches on every route
N_LARGE = 1 << 20      # docs of a sampled split
SCORE_ASC = [(ffi.SORT_SCORE, ffi.ORDER_ASC, ffi.ABSENT)]
DEEP_K = (4097, 8192, 10_000, 20_000)
FULL_HITS = 1          # QW_PLAN_FULL_HITS
MAPPING = {"field_mappings": [{"name": "body", "type": "text", "record": "freq", "fieldnorms": True},
                              {"name": "a", "type": "u64", "fast": True},
                              {"name": "c", "type": "u64", "fast": True},
                              {"name": "f", "type": "u64", "fast": True}]}


def cand_cap(K):
    return 8192 if K <= 4096 else (2 * K + 1023) // 1024 * 1024


def _hash(d, mul, mod):
    return (d.astype(np.uint64) * np.uint64(mul)) % np.uint64(mod)


class Corpus:
    """Arrays of one split: term frequencies of body terms (0 = absent), doc lengths, columns a, c and f."""

    def __init__(self, n, tf, lens, a, c, f, split_id):
        self.n, self.tf, self.lens, self.a, self.c, self.f = n, tf, lens, a, c, f
        b = S._Builder(n)
        L = ffi.img_lib()
        uniq, inv = np.unique(lens, return_inverse=True)
        fn = np.array([L.qwgpu_fieldnorm_to_id(int(x)) for x in uniq], dtype=np.uint8)[inv]
        body = b.add_field("body", ffi.FIELD_HAS_FREQS | ffi.FIELD_HAS_FIELDNORMS, ffi.TOK_DEFAULT, fn, int(lens.sum()))
        for name in sorted(tf):
            docs = np.flatnonzero(tf[name]).astype(np.uint32)
            b.add_term(body, name.encode(), docs, tf[name][docs].astype(np.uint32))
        for name, v in (("a", a), ("c", c), ("f", f)):
            b.add_column(name, ffi.COL_U64, ffi.CARD_FULL, v.astype(np.uint64), None)
        self.img = b.finish(split_id)
        self.norm = bm25_norm(lens)

    def scores(self, terms):
        """Union of `terms` in clause order in numpy float32, each term's weight checked against the compiled one."""
        s = np.zeros(self.n, dtype=np.float32)
        for t in terms:
            df = int(np.count_nonzero(self.tf[t]))
            w = np.float32(P.bm25_weight(df, self.n))
            assert abs(float(w) - float(bm25_weight(df, self.n))) <= 1e-6 * float(w)
            s = (s + bm25_contributions(self.tf[t], self.norm, w)).astype(np.float32)
        return s


def _benign(n, split_id, seed=0):
    d = np.arange(n, dtype=np.int64)
    present = (d % 16) != 15
    tf = {"x": 1 + (d * 13) % 15,
          "u": np.where(present, 1 + (d * 7 + seed) % 15, 0), "v": np.where(present, 1, 0),
          "w": np.where(present, 1 + (d * 11) % 15, 0), "z": np.where(d % 5 == 0, 1, 0),
          "rare": np.where(d % 97 == 3, 1, 0)}
    lens = 1 + _hash(d + seed, 7919, 400).astype(np.int64)
    a = _hash(d + 7 * seed, 2654435761, 1 << 32)
    return Corpus(n, tf, lens, a, _hash(d, 40503, 1000), d % 10, split_id)


# ---- routes: (query, sort, kernel bit, brute force) ------------------------------------------------------------------
CASES = ["union", "driver_col", "window_two_keys", "window_score_asc", "window_must_not"]
KERNEL = {"union": ffi.KERNEL_UNION, "driver_col": ffi.KERNEL_DRIVER, "window_two_keys": ffi.KERNEL_WINDOW,
          "window_score_asc": ffi.KERNEL_WINDOW, "window_must_not": ffi.KERNEL_WINDOW, "window_col": ffi.KERNEL_WINDOW}


def _should(img, *terms):
    return P.bool_([P.term(img, "body", t, occur=ffi.OCCUR_SHOULD) for t in terms])


def _plan(case, c, K, search_after=None):
    img = c.img
    root, sort = {
        "union": (_should(img, "u", "v"), SCORE_DESC),
        "driver_col": (P.bool_([P.term(img, "body", "x", occur=ffi.OCCUR_MUST), P.range_(img, "f", 0, 8, occur=ffi.OCCUR_FILTER)]),
                       [col_sort(img, "a", ffi.ORDER_DESC)]),
        "window_two_keys": (P.match_all(), [col_sort(img, "c", ffi.ORDER_DESC), col_sort(img, "a", ffi.ORDER_ASC)]),
        "window_score_asc": (_should(img, "w", "v"), SCORE_ASC),
        "window_must_not": (P.bool_([P.term(img, "body", "x", occur=ffi.OCCUR_MUST), P.term(img, "body", "z", occur=ffi.OCCUR_MUST_NOT)]),
                            [col_sort(img, "a", ffi.ORDER_DESC)]),
        "window_col": (P.match_all(), [col_sort(img, "a", ffi.ORDER_DESC)]),
    }[case]
    return P.make_plan(root, K, sort, search_after=search_after)


def _expected(case, c):
    """(matched docs in the sort's order, per-doc scores or None, second sort column or None)."""
    d = np.arange(c.n, dtype=np.int64)
    a, cc = c.a.astype(np.int64), c.c.astype(np.int64)
    sc, second = None, None
    if case == "union":
        m = (c.tf["u"] > 0) | (c.tf["v"] > 0)
        sc = c.scores(["u", "v"])
        keys = (-d, -sc)
    elif case == "window_score_asc":
        m = (c.tf["w"] > 0) | (c.tf["v"] > 0)
        sc = c.scores(["w", "v"])
        keys = (d, sc)
    elif case == "window_two_keys":
        m, keys, second = np.ones(c.n, dtype=bool), (-d, a, -cc), a
    elif case == "window_col":
        m, keys = np.ones(c.n, dtype=bool), (-d, -a)
    elif case == "window_must_not":
        m, keys = (c.tf["x"] > 0) & (c.tf["z"] == 0), (-d, -a)
    else:
        m, keys = (c.tf["x"] > 0) & (c.f <= 8), (-d, -a)
    docs = d[m]
    return docs[np.lexsort(tuple(k[m] for k in keys))], sc, second


def _check_brute(case, c, got, K, ctx, expected=None):
    order, sc, second = expected if expected is not None else _expected(case, c)
    want = order[:K]
    assert [h[0] for h in got.hits] == want.tolist(), f"{ctx}: doc ids differ from the brute force"
    if sc is not None:
        gs = np.array([h[4] for h in got.hits], dtype=np.float32).view(np.uint32)
        assert np.array_equal(gs, sc[want].view(np.uint32)), f"{ctx}: f32 score bits differ from the restatement"
    else:
        first = c.c if case == "window_two_keys" else c.a
        assert [h[2] for h in got.hits] == first[want].astype(np.int64).tolist(), f"{ctx}: sort values differ"
        if second is not None:
            assert [h[3] for h in got.hits] == c.a[want].astype(np.int64).tolist(), f"{ctx}: second sort values differ"
    assert got.num_hits == len(order)


def _path(r):
    return (f"kernel_mask={r.kernel_mask:#x} window_docs={r.window_docs} sample_stride={r.sample_stride} "
            f"exact_fallbacks={r.exact_fallbacks} refined={r.refined} radix_passes={r.radix_passes} launches={r.num_kernel_launches}")


def _run(ctx, case, c, K, label, search_after=None):
    pl = _plan(case, c, K, search_after)
    r = ctx.split_search([c.img.split_id], [pl])[0]
    tag = f"{label} {case} K={K}"
    print(f"[deep] {tag}: {_path(r)}")
    assert r.kernel_mask & KERNEL[case], f"{tag}: {_path(r)}"
    assert bool(r.kernel_mask & ffi.KERNEL_DEEP_SELECT) == (K > 4096), f"{tag}: {_path(r)}"
    assert_same(r, O.split_search(c.img, pl), ctx=tag)
    return r


@pytest.fixture(scope="module")
def small(gpu_ctx):
    c = _benign(N_SMALL, "deep-small")
    gpu_ctx.register_split(c.img)
    yield c
    gpu_ctx.unregister_split(c.img.split_id)


@pytest.mark.parametrize("case", CASES)
def test_routes(gpu_ctx, small, case):
    """Every route at K = 4096 (k_select) and above it (the deep path)."""
    exp = _expected(case, small)
    assert len(exp[0]) > 20_000
    for K in (4096,) + DEEP_K:
        r = _run(gpu_ctx, case, small, K, "route")
        _check_brute(case, small, r, K, f"route {case} K={K}", exp)
        assert len(r.hits) == K


def test_match_counts(gpu_ctx, small):
    """Fewer matches than K, and none."""
    img = small.img
    d = np.arange(small.n, dtype=np.int64)
    sort = [col_sort(img, "a", ffi.ORDER_DESC)]
    for K in (10_000, 20_000):
        pl = P.make_plan(P.bool_([P.term(img, "body", "rare", occur=ffi.OCCUR_MUST)]), K, sort)
        r = gpu_ctx.split_search([img.split_id], [pl])[0]
        assert r.kernel_mask & ffi.KERNEL_DEEP_SELECT, _path(r)
        assert_same(r, O.split_search(img, pl), ctx=f"rare K={K}")
        m = d[small.tf["rare"] > 0]
        want = m[np.argsort(-small.a[m].astype(np.int64), kind="stable")]
        assert len(m) < K and [h[0] for h in r.hits] == want.tolist() and r.num_hits == len(m)
        pl = P.make_plan(P.bool_([P.term(img, "body", "x", occur=ffi.OCCUR_MUST), P.range_(img, "f", 50, 60, occur=ffi.OCCUR_FILTER)]), K, sort)
        r = gpu_ctx.split_search([img.split_id], [pl])[0]
        assert r.num_hits == 0 and r.hits == [], _path(r)
        assert_same(r, O.split_search(img, pl), ctx=f"none K={K}")


def test_search_after(gpu_ctx, small):
    order, _, _ = _expected("window_col", small)
    for rank in (5, 3000, 9000):
        marker = int(order[rank])
        sa = ffi.QwSearchAfter(1, 1, 0, 1, 0, marker, int(small.a[marker]), 0)
        for K in (4097, 10_000):
            r = _run(gpu_ctx, "window_col", small, K, f"search_after@{rank}", search_after=sa)
            assert [h[0] for h in r.hits] == order[rank + 1: rank + 1 + K].tolist()
            assert r.num_hits == len(order)


# ---- ties on the first key word ------------------------------------------------------------------------------------------
def _tie_split(n, split_id, above, tie):
    """Column g: `above` docs above the tie value, `tie` docs on it, every other doc below; two 60-bit sort columns
    keep the doc id out of the first key word, and column b (few values) orders within the tie, the doc id last."""
    d = np.arange(n, dtype=np.int64)
    b = S._Builder(n)
    fid = b.add_field("body", ffi.FIELD_HAS_FREQS | ffi.FIELD_HAS_FIELDNORMS, ffi.TOK_DEFAULT, np.full(n, 1, np.uint8), n)
    b.add_term(fid, b"x", np.arange(n, dtype=np.uint32), np.ones(n, dtype=np.uint32))
    tie_v = (1 << 59)
    g = _hash(d, 2654435761, 1 << 40)   # below the tie
    pick = np.random.default_rng(7).permutation(n)
    g[pick[:above]] = tie_v + 1 + _hash(d[pick[:above]], 40503, 1 << 40)
    g[pick[above:above + tie]] = tie_v
    bb = (d % 7).astype(np.uint64)
    bb[0] = (1 << 60) - 1
    b.add_column("g", ffi.COL_U64, ffi.CARD_FULL, g, None)
    b.add_column("b", ffi.COL_U64, ffi.CARD_FULL, bb, None)
    return b.finish(split_id), g, bb


@pytest.mark.parametrize("above, tie, K", [(8_500, 3_000, 10_000), (3_000, 3_000, 4_500), (0, 25_000, 10_000), (100, 25_000, 20_000)])
def test_ties(gpu_ctx, above, tie, K):
    """A ~3000-doc tie on the first key word straddling the K-th hit (it spans 2048-survivor tiles), and a top-key tie
    larger than the candidate capacity, which the exact radix descent resolves down to the doc id."""
    n = 200_000
    img, g, bb = _tie_split(n, f"deep-ties-{above}-{tie}", above, tie)
    gpu_ctx.register_split(img)
    try:
        pl = P.make_plan(P.match_all(), K, [col_sort(img, "g", ffi.ORDER_DESC), col_sort(img, "b", ffi.ORDER_ASC)])
        r = gpu_ctx.split_search([img.split_id], [pl])[0]
        print(f"[deep] ties above={above} tie={tie} K={K}: {_path(r)}")
        assert r.kernel_mask & ffi.KERNEL_DEEP_SELECT and r.kernel_mask & ffi.KERNEL_WINDOW, _path(r)
        if above + tie > cand_cap(K):
            assert r.radix_passes > 0, _path(r)
        assert_same(r, O.split_search(img, pl), ctx=f"ties {above}/{tie} K={K}")
        d = np.arange(n, dtype=np.int64)
        want = np.lexsort((-d, bb.astype(np.uint64), ~g.astype(np.uint64)))[:K]
        assert [h[0] for h in r.hits] == want.tolist()
        assert [h[2] for h in r.hits] == g[want].tolist() and [h[3] for h in r.hits] == bb[want].tolist()
    finally:
        gpu_ctx.unregister_split(img.split_id)


# ---- the sampled threshold at deep K ---------------------------------------------------------------------------------------
SAMPLED = ["union", "window_col", "driver_col"]


@pytest.fixture(scope="module")
def large(gpu_ctx):
    c = _benign(N_LARGE, "deep-large")
    gpu_ctx.register_split(c.img)
    yield c
    gpu_ctx.unregister_split(c.img.split_id)


@pytest.fixture(scope="module")
def probe(gpu_ctx, large):
    """(window_docs, sample_stride) of every sampled case on the 1 M-doc split, read back from the engine."""
    out = {}
    for case in SAMPLED:
        r = gpu_ctx.split_search([large.img.split_id], [_plan(case, large, 10)])[0]
        assert r.sample_stride >= 3, f"{case}: {_path(r)}"
        out[case] = (r.window_docs, r.sample_stride)
    return out


# K at which the benign corpus's sample holds. The sample's target (2K/stride + 24, k_pick) keeps about 2K + 24 * stride
# candidates plus the rest of the threshold's 11-bit digit bin (~N/2048 keys of a uniform column, far more for BM25
# scores of few distinct values), and the capacity leaves 2K rounded up to 1024: at K = 4097 that room is 1022 keys,
# enough for the uniform column on k_window (stride 4) and k_driver (stride 16). Elsewhere the candidates may
# overshoot the capacity and the call is repaired, exactly.
SAMPLE_HOLDS = {"union": (), "window_col": (4097,), "driver_col": (4097,)}


@pytest.mark.parametrize("case", SAMPLED)
def test_sample_passes(gpu_ctx, large, probe, case):
    """Benign keys on a 1 M-doc split: the deep path after a sampled threshold, with or without its repair."""
    exp = _expected(case, large)
    for K in (4097, 10_000, 20_000):
        r = _run(gpu_ctx, case, large, K, "sampled")
        _check_brute(case, large, r, K, f"sampled {case} K={K}", exp)
        assert r.sample_stride >= 3 and r.exact_fallbacks <= 1, _path(r)
        if K in SAMPLE_HOLDS[case]:
            assert r.exact_fallbacks == 0 and r.radix_passes == 0 and r.refined == 0, _path(r)
        elif r.exact_fallbacks:
            assert r.refined == (1 if case == "window_col" else 0), _path(r)


def _h(K, s):
    """Top keys in one sampled window so that the sample alone reaches its target rank (see k_pick)."""
    return -(-2 * K // s) + 24 + 16


def _adversarial(n, W, s, scenario, K, tie, split_id):
    """scenario "high": class 3 = _h(K, s) docs at the start of window s (sampled), class 2 = every doc of windows
    1..s-1 (never sampled), class 1 = the rest. scenario "low": class 3 = `tie` docs with one and the same top key,
    all but two in windows no sample reads."""
    d = np.arange(n, dtype=np.int64)
    win = d // W
    nw = (n + W - 1) // W
    cls = np.ones(n, dtype=np.int64)
    if scenario == "high":
        assert 3 <= s and s + 1 < nw and _h(K, s) < K and _h(K, s) <= W and (s - 1) * W >= K
        cls[(win >= 1) & (win < s)] = 2
        cls[s * W: s * W + _h(K, s)] = 3
    else:
        unsampled = np.flatnonzero((win % s != 0) & (win != 0) & (win != nw - 1))
        cls[unsampled[np.linspace(0, len(unsampled) - 1, tie - 2).astype(np.int64)]] = 3
        cls[[s * W + 1, s * W + 5]] = 3
    present = ((d % 16) != 15) | (cls > 1)
    up = np.array([0, 1, 2, 15])[cls]
    tf = {"x": up, "u": np.where(present, up, 0), "v": np.where(present, 1, 0), "w": np.where(present, 1, 0),
          "z": np.zeros(n, dtype=np.int64), "rare": np.where(d % 97 == 3, 1, 0)}
    lens = np.where((cls == 3) & (scenario == "low"), 10, 8 + d % 5)
    r = _hash(d, 2654435761, 1 << 20).astype(np.int64)
    a = np.where(cls == 3, (0xFFFFFFFF if scenario == "low" else 0xC0000000 + r), np.where(cls == 2, 0x40000000 + r, r))
    f = np.where(cls > 1, 0, d % 10)
    return Corpus(n, tf, lens, a, _hash(d, 40503, 1000), f, split_id)


# (k_driver samples 128-doc posting blocks: the ~1300 top keys that lift its sample too high at K = 10 000 do not fit one)
@pytest.mark.parametrize("case, scenario", [("union", "high"), ("window_col", "high"),
                                            ("union", "low"), ("window_col", "low"), ("driver_col", "low")])
def test_sample_fails(gpu_ctx, probe, case, scenario):
    """Too high: the K-th key lies in windows the sample never read. Too low: the top key repeats on more docs than the
    candidate capacity (25 000 against 20 480 at K = 10 000). Column sorts with the level-0 histogram on record take the candidates-only repair; `_score`
    sorts and the posting-driven kernel re-run the exact radix descent."""
    K = 10_000
    W, s = probe[case]
    c = _adversarial(N_LARGE, W, s, scenario, K, 25_000, f"deep-{scenario}-{case}")
    gpu_ctx.register_split(c.img)
    try:
        r = _run(gpu_ctx, case, c, K, f"too-{scenario}")
        assert r.sample_stride >= 3 and r.exact_fallbacks == 1 and r.radix_passes >= 1, _path(r)
        assert r.refined == (1 if case == "window_col" else 0), _path(r)
        _check_brute(case, c, r, K, f"too-{scenario} {case}")
        if scenario == "high":
            assert 1 <= r.hits[K - 1][0] // W < s, "the K-th hit lies in a window the sample never read"
    finally:
        gpu_ctx.unregister_split(c.img.split_id)


# ---- record layout and batches -------------------------------------------------------------------------------------------
def _with_full_hits(plan):
    h = ffi.QwPlanHeader.from_buffer_copy(plan)
    h.reserved |= FULL_HITS
    return bytes(h) + plan[C.sizeof(h):]


def _raw_search(ctx, ids, plans):
    """Seam C, keeping each split's QwHit array as raw bytes and the call's kernel mask."""
    L = ffi.lib()
    n = len(ids)
    bufs = [C.create_string_buffer(p, len(p)) for p in plans]
    res = (ffi.SplitResult * n)()
    status = (C.c_int * n)()
    ffi.check(L.qwgpu_split_search(ctx._ctx, n, (C.c_char_p * n)(*[s.encode() for s in ids]),
                                   (C.c_void_p * n)(*[C.addressof(b) for b in bufs]), (C.c_size_t * n)(*[len(p) for p in plans]),
                                   res, status))
    try:
        assert list(status) == [0] * n, L.qwgpu_last_error().decode()
        return [C.string_at(res[i].hits, res[i].num_partial_hits * C.sizeof(ffi.QwHit)) for i in range(n)], res[0].kernel_mask
    finally:
        for i in range(n):
            L.qwgpu_split_result_free(C.byref(res[i]))


@pytest.fixture(scope="module")
def twins(gpu_ctx):
    cs = [_benign(N_SMALL, f"deep-twin-{i}", seed=i + 1) for i in range(2)]
    for c in cs:
        gpu_ctx.register_split(c.img)
    yield cs
    for c in cs:
        gpu_ctx.unregister_split(c.img.split_id)


def test_compact_hits_equal_full_records(gpu_ctx, small, twins):
    """A deep `_score` plan returns (doc id, score) pairs expanded on the host: the same bytes as full records."""
    cs = [small] + twins
    ids = [c.img.split_id for c in cs]
    for K in (4097, 10_000, 20_000):
        plans = [_plan("union", c, K) for c in cs]
        got, mask = _raw_search(gpu_ctx, ids, plans)
        want, wmask = _raw_search(gpu_ctx, ids, [_with_full_hits(p) for p in plans])
        assert mask == wmask and mask & ffi.KERNEL_DEEP_SELECT and mask & ffi.KERNEL_UNION, hex(mask)
        for i, (g, w) in enumerate(zip(got, want)):
            assert len(g) == K * C.sizeof(ffi.QwHit) and g == w, f"K={K} split {i}: QwHit bytes differ"


@pytest.mark.parametrize("case", ["union", "window_two_keys"])
def test_mixed_batch(gpu_ctx, small, twins, case):
    """One call with a K = 1000 split and K = 10 000 splits: the shallow split's hits are the bytes it gets alone."""
    cs = [twins[0], small, twins[1]]
    Ks = [1000, 10_000, 10_000]
    got, mask = _raw_search(gpu_ctx, [c.img.split_id for c in cs], [_plan(case, c, K) for c, K in zip(cs, Ks)])
    assert mask & ffi.KERNEL_DEEP_SELECT, hex(mask)
    alone, amask = _raw_search(gpu_ctx, [twins[0].img.split_id], [_plan(case, twins[0], 1000)])
    assert not amask & ffi.KERNEL_DEEP_SELECT, hex(amask)
    assert got[0] == alone[0], "the shallow split's hits differ in a batch with deep splits"
    for c, K, raw in zip(cs[1:], Ks[1:], got[1:]):
        h = np.frombuffer(raw, dtype=np.dtype([("v1", "<u8"), ("v2", "<u8"), ("doc_id", "<u4"), ("flags", "<u4"),
                                               ("score", "<f4"), ("reserved", "<u4")]))
        assert h["doc_id"].tolist() == _expected(case, c)[0][:K].tolist()


# ---- qwgpu_leaf_search: per-split deep lists merged on the device ---------------------------------------------------------
@pytest.fixture(scope="module")
def leaf_splits(gpu_ctx):
    cs = [_benign(40_000, f"deep-leaf-{i}", seed=i) for i in range(8)]
    for c in cs:
        gpu_ctx.register_split(c.img)
    yield cs
    for c in cs:
        gpu_ctx.unregister_split(c.img.split_id)


@pytest.mark.parametrize("sort", ["_score", "a"])
@pytest.mark.parametrize("start, max_hits", [(0, 10_000), (10_000, 10_000), (4000, 200)])
def test_leaf_search(gpu_ctx, leaf_splits, sort, start, max_hits):
    imgs = [c.img for c in leaf_splits]
    ast = bool_(should=[term("body", "u"), term("body", "v")])
    kw = dict(max_hits=max_hits, start_offset=start, sort_fields=[(sort, proto.DESC)])
    offsets = [proto.enc_split_offsets(im.split_id, im.num_docs) for im in imgs]
    lreq = proto.enc_leaf_search_request(search_request(ast, **leafify(kw)), offsets, json.dumps(MAPPING))
    got = proto.dec_leaf_search_response(service.merge_leaf_responses(search_request(ast, **kw), [gpu_ctx.leaf_search(lreq)]))
    want = cpu_root_search(imgs, ast, MAPPING, **kw)
    assert got["num_hits"] == want["num_hits"]
    assert len(got["partial_hits"]) == max_hits
    assert got["partial_hits"] == want["partial_hits"]


def test_refuses_more_than_20000_hits(gpu_ctx, small):
    pl = _plan("union", small, 20_001)
    with pytest.raises(ffi.QwGpuError) as e:
        gpu_ctx.split_search([small.img.split_id], [pl])
    assert e.value.code == ffi.EUNSUPPORTED and "20 000" in e.value.msg


# ---- the context's limit, through qwgpu_leaf_search and seam C ------------------------------------------------------------------
SYNTH_MAPPING = {"field_mappings": [{"name": "body", "type": "text", "record": "freq", "fieldnorms": True},
                                    {"name": "severity_text", "type": "text", "tokenizer": "raw", "fast": True},
                                    {"name": "timestamp", "type": "datetime", "fast": True, "fast_precision": "seconds"},
                                    {"name": "tenant_id", "type": "u64", "fast": True}], "timestamp_field": "timestamp"}


@pytest.fixture(scope="module")
def synth(gpu_ctx):
    img = S.synth_split(40_000, 0, [0.2, 0.1, 0.05], split_id="deep-synth-0", ts_start_secs=1_700_000_000)
    gpu_ctx.register_split(img)
    yield [img]
    gpu_ctx.unregister_split(img.split_id)


def _leaf(ctx, img, max_hits):
    offsets = [proto.enc_split_offsets(img.split_id, img.num_docs)]
    req = proto.enc_leaf_search_request(search_request(term("body", "t0"), max_hits=max_hits), offsets, json.dumps(SYNTH_MAPPING))
    return proto.dec_leaf_search_response(ctx.leaf_search(req))


def test_limit_through_leaf_search(gpu_ctx, synth):
    """A request above the context's limit fails the same way on every node: the split is reported failed but NOT
    retryable, so the root does not run it twice. The default limit is 4096; raised, 5000 hits are served and 20 001
    stay refused."""
    img = synth[0]

    def refused(resp):
        assert resp["num_successful_splits"] == 0 and len(resp["failed_splits"]) == 1, resp["failed_splits"]
        f = resp["failed_splits"][0]
        assert f["retryable_error"] is False and f["split_id"] == img.split_id
        return f["error"]

    gpu_ctx.set_max_hits(4096)
    try:
        assert "qwgpu_set_max_hits" in refused(_leaf(gpu_ctx, img, 5000))
        assert len(_leaf(gpu_ctx, img, 4096)["partial_hits"]) == 4096
    finally:
        gpu_ctx.set_max_hits(20_000)
    resp = _leaf(gpu_ctx, img, 5000)
    assert resp["num_successful_splits"] == 1 and len(resp["partial_hits"]) == 5000
    assert "20 000" in refused(_leaf(gpu_ctx, img, 20_001))


def test_limit_bounds(gpu_ctx, small):
    for bad in (0, 20_001):
        with pytest.raises(ffi.QwGpuError) as e:
            gpu_ctx.set_max_hits(bad)
        assert e.value.code == ffi.EINVALID_ARG
    gpu_ctx.set_max_hits(4096)
    try:
        with pytest.raises(ffi.QwGpuError) as e:
            gpu_ctx.split_search([small.img.split_id], [_plan("union", small, 4097)])
        assert e.value.code == ffi.EUNSUPPORTED
        r = gpu_ctx.split_search([small.img.split_id], [_plan("union", small, 4096)])[0]
        assert len(r.hits) == 4096 and not r.kernel_mask & ffi.KERNEL_DEEP_SELECT
    finally:
        gpu_ctx.set_max_hits(20_000)
