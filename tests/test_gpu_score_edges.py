"""`_score` top-K with the K-th key on a bucket edge of the composite key, on every route (DESIGN.md §4.6).

The corpora (score_edges_ref.EdgeCorpus) plant docs exactly on an integer x = fmul(score, score_scale), 1..8 ulps above
it (inside the band the float bounds of k_union and k_window's fast path leave below a bucket), 1..8 ulps below it, in
the clamped bucket 1023 (x = 1024 at score == score_max) and in bucket 0 (a union whose boosts differ by 1000x). Each
call asserts the path it took and is checked bit for bit against the brute force over the corpus arrays (doc ids, f32
score bits, num_hits) and against the oracle. Where the sampled threshold is expected to hold, `exact_fallbacks == 0`
is asserted too: a repair would hide a doc that the sampled pass dropped."""
import numpy as np
import pytest

from quickwit_b200 import ffi, plan as P, splitgen as S
from oracle import oracle as O
from helpers import SCORE_DESC, assert_same
import score_edges_ref as R

pytestmark = pytest.mark.gpu

N_BIG = 2_100_000      # 137 k_union windows: a sampled threshold alone, the fused sample under nine ids
N_SMALL = 200_000      # 14 windows: no sample, the exact radix descent
N_IDS = 9
SCORE_ASC = [(ffi.SORT_SCORE, ffi.ORDER_ASC, ffi.ABSENT)]
# (edge term, K, ulps of the K-th hit's x from the edge)
EDGES = [("e1", 1, 8), ("e10", 10, 0), ("e1000", 1000, None), ("e4096", 4096, 0)]


def _path(r):
    return (f"kernel_mask={r.kernel_mask:#x} window_docs={r.window_docs} sample_stride={r.sample_stride} "
            f"launches={r.num_kernel_launches} exact_fallbacks={r.exact_fallbacks} refined={r.refined} "
            f"radix_passes={r.radix_passes}")


def _clauses(img, clauses, must_not=()):
    kids = [P.term(img, "body", t, occur=ffi.OCCUR_SHOULD, boost=b) for t, b in clauses]
    kids += [P.term(img, "body", t, occur=ffi.OCCUR_MUST_NOT) for t in must_not]
    return P.bool_(kids)


def _expected(c, clauses, must_not=(), desc=True, extra=None):
    s = c.scores(clauses)
    m = np.zeros(c.n, dtype=bool)
    for t, _ in clauses:
        m |= c.tf[t] > 0
    for t in must_not:
        m &= c.tf[t] == 0
    if extra is not None:
        m &= extra
    return R.brute_order(s, m, desc), s


def _check(c, r, pl, want, s, K, tag, skip=0):
    order = want[skip: skip + K]
    assert [h[0] for h in r.hits] == order.tolist(), f"{tag}: doc ids differ from the brute force ({_path(r)})"
    got = np.array([h[4] for h in r.hits], dtype=np.float32).view(np.uint32)
    assert np.array_equal(got, s[order].view(np.uint32)), f"{tag}: f32 score bits differ"
    assert r.num_hits == len(want), f"{tag}: num_hits"
    assert_same(r, O.split_search(c.img, pl), ctx=tag)


def _run(ctx, c, root, K, sort=SCORE_DESC, search_after=None):
    pl = P.make_plan(root, K, sort, search_after=search_after)
    return ctx.split_search([c.img.split_id], [pl])[0], pl


def _sampled_and_skipped(c, t, r):
    """The edge classes of term t lie both in windows the call's sample read and in windows it skipped, from the window
    size and stride the engine reports (a split at batch position 0 samples windows 0, stride, 2 stride, ...)."""
    assert r.window_docs > 0 and r.sample_stride >= 2, _path(r)
    for k in ("above", "exact", "below"):
        docs = c.planted[t][k]
        if len(docs) < 32:
            continue
        sampled = (docs // r.window_docs) % r.sample_stride == 0
        assert sampled.any() and (~sampled).any(), f"{t} {k}: {_path(r)}"


def _kth_ulps(c, t, s, want, K):
    return int(R.ulps_from(R.fmul(s[want[K - 1]], c.scale(c.clauses(t))), c.l[t]))


@pytest.fixture(scope="module")
def small(gpu_ctx):
    c = R.EdgeCorpus(N_SMALL, "edges-small")
    gpu_ctx.register_split(c.img)
    yield c
    gpu_ctx.unregister_split(c.img.split_id)


@pytest.fixture(scope="module")
def big(gpu_ctx):
    c = R.EdgeCorpus(N_BIG, "edges-big")
    gpu_ctx.register_split(c.img)
    yield c
    gpu_ctx.unregister_split(c.img.split_id)


@pytest.mark.parametrize("t,K,ulps", EDGES)
def test_union_exact(gpu_ctx, small, t, K, ulps):
    """k_union without a sample: the threshold is the exact bucket of the K-th key, so a bound that drops a doc of
    that bucket leaves fewer than K candidates."""
    c = small
    want, s = _expected(c, c.clauses(t))
    if ulps is not None:
        assert _kth_ulps(c, t, s, want, K) == ulps
    else:
        assert -R.BAND <= _kth_ulps(c, t, s, want, K) < 0
    for k in (K, K + 1) if K == 4096 else (K,):   # 4097: the deep selection path, past the context's default limit
        if k > 4096:
            gpu_ctx.set_max_hits(k)
        try:
            r, pl = _run(gpu_ctx, c, _clauses(c.img, c.clauses(t)), k)
        finally:
            if k > 4096:
                gpu_ctx.set_max_hits(4096)
        print(f"[edges] union exact {t} K={k}: {_path(r)}")
        assert r.kernel_mask & ffi.KERNEL_UNION and r.sample_stride == 0 and r.radix_passes >= 1, _path(r)
        assert r.exact_fallbacks == 0 and r.refined == 0, _path(r)
        assert bool(r.kernel_mask & ffi.KERNEL_DEEP_SELECT) == (k > 4096), _path(r)
        _check(c, r, pl, want, s, k, f"union exact {t} K={k}")


@pytest.mark.parametrize("t,K,ulps", EDGES[:3])
def test_union_sampled(gpu_ctx, big, t, K, ulps):
    """k_union's separate sampled pass: the sample must pick the edge bucket (its histogram digit agrees with the key)
    and the sweep's float bound must keep every doc of it."""
    c = big
    want, s = _expected(c, c.clauses(t))
    r, pl = _run(gpu_ctx, c, _clauses(c.img, c.clauses(t)), K)
    print(f"[edges] union sampled {t} K={K}: {_path(r)}")
    assert r.kernel_mask & ffi.KERNEL_UNION and r.sample_stride >= 2, _path(r)
    assert r.exact_fallbacks == 0 and r.radix_passes == 0 and r.refined == 0, _path(r)
    _sampled_and_skipped(c, t, r)
    _check(c, r, pl, want, s, K, f"union sampled {t} K={K}")


def test_union_fused_sample(gpu_ctx, big):
    """k_union<MODE_SAMPLE_COLLECT>: the same split under nine ids, each block sampling its first window."""
    twins = [big] + [big.under_id(f"edges-big-{i}") for i in range(1, N_IDS)]
    for c in twins[1:]:
        gpu_ctx.register_split(c.img)
    try:
        for t, K, _ in EDGES[:3]:
            plans = [P.make_plan(_clauses(c.img, c.clauses(t)), K, SCORE_DESC) for c in twins]
            res = gpu_ctx.split_search([c.img.split_id for c in twins], plans)
            print(f"[edges] fused {t} K={K}: {_path(res[0])}")
            assert res[0].num_kernel_launches == 2 and res[0].exact_fallbacks == 0, _path(res[0])
            want, s = _expected(big, big.clauses(t))
            for i in (0, N_IDS - 1):
                _check(twins[i], res[i], plans[i], want, s, K, f"fused {t} K={K} split {i}")
    finally:
        for c in twins[1:]:
            gpu_ctx.unregister_split(c.img.split_id)


@pytest.mark.parametrize("which", ["small", "big"])
def test_window_fast_path(gpu_ctx, small, big, which):
    """k_window's BM25 fast path: the union carries a must_not, so it leaves k_union."""
    c = small if which == "small" else big
    for t, K, _ in EDGES[:3] + ([EDGES[3]] if which == "small" else []):
        want, s = _expected(c, c.clauses(t), must_not=("x",))
        r, pl = _run(gpu_ctx, c, _clauses(c.img, c.clauses(t), must_not=("x",)), K)
        print(f"[edges] window fast {which} {t} K={K}: {_path(r)}")
        assert r.kernel_mask & ffi.KERNEL_WINDOW and not r.kernel_mask & ffi.KERNEL_UNION, _path(r)
        assert (r.sample_stride >= 2) == (which == "big"), _path(r)
        assert r.exact_fallbacks == 0 and r.refined == 0, _path(r)
        if which == "big":
            _sampled_and_skipped(c, t, r)
        else:
            assert r.radix_passes >= 1, _path(r)
        _check(c, r, pl, want, s, K, f"window fast {which} {t} K={K}")


def test_window_fast_path_in_a_mixed_batch(gpu_ctx, small):
    """A pure OR batched with a driver plan: the batch runs on k_window, the OR on its fast path."""
    c = small
    t, K, _ = EDGES[1]
    twin = c.under_id("edges-small-twin")
    gpu_ctx.register_split(twin.img)
    plans = [P.make_plan(_clauses(c.img, c.clauses(t)), K, SCORE_DESC),
             P.make_plan(P.bool_([P.term(c.img, "body", "top"), P.range_(c.img, "f", 0, 0)]), 10, SCORE_DESC)]
    try:
        res = gpu_ctx.split_search([c.img.split_id, twin.img.split_id], plans)
    finally:
        gpu_ctx.unregister_split(twin.img.split_id)
    print(f"[edges] mixed batch: {_path(res[0])}")
    assert res[0].kernel_mask & ffi.KERNEL_WINDOW and not res[0].kernel_mask & ffi.KERNEL_UNION, _path(res[0])
    assert res[0].sample_stride >= 2 and res[0].exact_fallbacks == 0 and res[0].refined == 0, _path(res[0])
    want, s = _expected(c, c.clauses(t))
    _check(c, res[0], plans[0], want, s, K, "mixed batch")


@pytest.mark.parametrize("which", ["small", "big"])
def test_window_score_asc(gpu_ctx, small, big, which):
    """k_window generic, `_score` ASC: digit 1023 - lin; the lowest scores sit 1..8 ulps below the edge, then the tie
    on it."""
    c = small if which == "small" else big
    want, s = _expected(c, c.clauses("asc"), desc=False)
    for K, lo, hi in ((10, -R.BAND, -1), (1000, 0, 0)):
        assert lo <= _kth_ulps(c, "asc", s, want, K) <= hi
        r, pl = _run(gpu_ctx, c, _clauses(c.img, c.clauses("asc")), K, sort=SCORE_ASC)
        print(f"[edges] window asc {which} K={K}: {_path(r)}")
        assert r.kernel_mask & ffi.KERNEL_WINDOW and not r.kernel_mask & ffi.KERNEL_UNION, _path(r)
        assert (r.sample_stride >= 2) == (which == "big"), _path(r)
        assert r.exact_fallbacks == 0 and r.refined == 0, _path(r)
        if which == "big":
            _sampled_and_skipped(c, "asc", r)
        else:
            assert r.radix_passes >= 1, _path(r)
        _check(c, r, pl, want, s, K, f"window asc {which} K={K}")


def test_window_search_after_inside_the_band(gpu_ctx, big):
    """k_window generic, `_score` DESC with search_after: the page starts inside the edge's band and inside its tie."""
    c = big
    t = "e1000"
    want, s = _expected(c, c.clauses(t))
    for rank, K in ((200, 1000), (700, 10)):   # (a doc 1..8 ulps above the edge; a doc of the tie on it)
        marker = int(want[rank])
        sa = ffi.QwSearchAfter(1, 1, 0, 1, 0, marker, S.f64_to_u64(float(s[marker])), 0)
        r, pl = _run(gpu_ctx, c, _clauses(c.img, c.clauses(t)), K, search_after=sa)
        print(f"[edges] search_after@{rank} K={K}: {_path(r)}")
        assert r.kernel_mask & ffi.KERNEL_WINDOW and not r.kernel_mask & ffi.KERNEL_UNION, _path(r)
        assert r.sample_stride >= 2 and r.exact_fallbacks == 0 and r.refined == 0 and r.radix_passes == 0, _path(r)
        assert [h[0] for h in r.hits] == want[rank + 1: rank + 1 + K].tolist(), f"search_after@{rank}"
        got = np.array([h[4] for h in r.hits], dtype=np.float32).view(np.uint32)
        assert np.array_equal(got, s[want[rank + 1: rank + 1 + K]].view(np.uint32))
        assert_same(r, O.split_search(c.img, pl), ctx=f"search_after@{rank}")


@pytest.mark.parametrize("which", ["small", "big"])
def test_driver_clamped_bucket(gpu_ctx, small, big, which):
    """k_driver, scored term AND range filter: score_max is the term's weight, so docs at tf 2^32 - 1 score it whole and
    land on x = 1024, clamped into bucket 1023 together with the docs around x = 1023."""
    c = small if which == "small" else big
    keep = c.f <= 0
    want, s = _expected(c, [("top", 1.0)], extra=keep)
    root = P.bool_([P.term(c.img, "body", "top"), P.range_(c.img, "f", 0, 0)])
    for K in (10, 50):
        r, pl = _run(gpu_ctx, c, root, K)
        print(f"[edges] driver {which} K={K}: {_path(r)}")
        # (`top` holds 240 docs, two posting blocks: too few to sample, so the exact descent runs)
        assert r.kernel_mask & ffi.KERNEL_DRIVER and r.sample_stride == 0 and r.radix_passes >= 1, _path(r)
        assert r.exact_fallbacks == 0 and r.refined == 0, _path(r)
        assert R.lin(s[want[K - 1]], c.scale([("top", 1.0)])) == 1023
        _check(c, r, pl, want, s, K, f"driver {which} K={K}")


@pytest.mark.parametrize("must_not", [(), ("x",)])
def test_bucket_zero(gpu_ctx, small, must_not):
    """A union whose boosts differ by 1000x: the K-th key of `tune_e1^1000 OR g` is in bucket 0, where k_union's bound
    and k_window's fast-path bound (-inf) must both keep every match."""
    c = small
    clauses = [("tune_e1", 1000.0), ("g", 1.0)]
    K = 1000
    want, s = _expected(c, clauses, must_not=must_not)
    assert R.lin(s[want[K - 1]], c.scale(clauses)) == 0
    r, pl = _run(gpu_ctx, c, _clauses(c.img, clauses, must_not=must_not), K)
    print(f"[edges] bucket 0 must_not={must_not}: {_path(r)}")
    assert r.kernel_mask & (ffi.KERNEL_WINDOW if must_not else ffi.KERNEL_UNION), _path(r)
    # (bucket 0 holds ~25 000 matches: the exact descent goes past level 0)
    assert r.sample_stride == 0 and r.radix_passes >= 2 and r.exact_fallbacks == 0 and r.refined == 0, _path(r)
    _check(c, r, pl, want, s, K, f"bucket 0 must_not={must_not}")


@pytest.mark.parametrize("route", ["exact", "sampled", "fused"])
def test_union_clamped_bucket(gpu_ctx, small, big, route):
    """k_union on `ca OR cb` with docs at both clauses' tf 2^32 - 1: they score score_max exactly, x = 1024, and only the
    clamp keeps their digit in bucket 1023, on the sample histogram (`score_digit`) as in the key (`score_lin`). The
    K-th key lies in that bucket; far below it one bucket holds a 9000-doc tie, so a sample that lost bucket 1023 would
    pick that bucket and overflow the candidate capacity."""
    c = small if route == "exact" else big
    cl = c.clamp_clauses()
    want, s = _expected(c, cl)
    scale = c.scale(cl)
    smax = np.float32(c.weight(*cl[0]) + c.weight(*cl[1]))
    splits = [c] if route != "fused" else [c] + [c.under_id(f"edges-big-clamp-{i}") for i in range(1, N_IDS)]
    for t in splits[1:]:
        gpu_ctx.register_split(t.img)
    try:
        for K in (10, 1000):
            assert s[want[K - 1]] == smax and R.fmul(s[want[K - 1]], scale) == 1024 and R.lin(s[want[K - 1]], scale) == 1023
            plans = [P.make_plan(_clauses(t.img, cl), K, SCORE_DESC) for t in splits]
            res = gpu_ctx.split_search([t.img.split_id for t in splits], plans)
            r = res[0]
            print(f"[edges] clamp {route} K={K}: {_path(r)}")
            assert r.kernel_mask & ffi.KERNEL_UNION and r.exact_fallbacks == 0 and r.refined == 0, _path(r)
            if route == "exact":
                assert r.sample_stride == 0 and r.radix_passes >= 1, _path(r)
            elif route == "sampled":
                assert r.sample_stride >= 2 and r.radix_passes == 0 and r.num_kernel_launches > 2, _path(r)
            else:
                assert r.num_kernel_launches == 2 and r.radix_passes == 0, _path(r)
            for i in (0, len(splits) - 1):
                _check(splits[i], res[i], plans[i], want, s, K, f"clamp {route} K={K} split {i}")
    finally:
        for t in splits[1:]:
            gpu_ctx.unregister_split(t.img.split_id)
