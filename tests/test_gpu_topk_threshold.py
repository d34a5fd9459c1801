"""The sampled top-K threshold and its two repairs, on every kernel that samples (DESIGN.md §4.6).

A top-K query over a split with enough windows first estimates its threshold from a 1/stride sample of the windows
(k_driver: of the driving term's posting blocks), collects with it and checks the candidate count of every split. A
failed check is repaired by a candidates-only pass over the failing splits (column and doc-id sorts) or by an exact
radix descent from level 0 (`_score` sorts). Test corpora of ~1 M docs per split reach the sampled path; the keys are
placed from the window size and stride the engine reports (`window_docs`, `sample_stride`) so that the sample
  * passes (benign keys),
  * is too high: a few top keys sit in a sampled window, the rest of the top K in windows no sample reads,
  * is too low: the top value repeats over more docs than the candidate capacity, almost all of them unsampled.
Every result is checked bit for bit against the oracle AND against a brute force over the arrays the corpus was
generated from (numpy lexsort for column sorts, the numpy float32 BM25 restatement for `_score` sorts), and the path
the call took is asserted from the result's kernel_mask / sample_stride / exact_fallbacks / refined / radix_passes."""
import json

import numpy as np
import pytest

from quickwit_b200 import ffi, plan as P, proto, service, splitgen as S
from oracle import oracle as O
from helpers import SCORE_DESC, assert_same, bm25_contributions, bm25_norm, bm25_weight, col_sort
from pipeline import bool_, cpu_root_search, leafify, search_request, term

pytestmark = pytest.mark.gpu

N = 1 << 20          # docs per large split: >= 16 windows (or 1024 driving blocks) on every kernel
CAND_CAP = 8192      # QW_CAND_CAP
TIE = 10_000         # > CAND_CAP docs sharing the top key
MAPPING = {"field_mappings": [{"name": "body", "type": "text", "record": "freq", "fieldnorms": True},
                              {"name": "a", "type": "u64", "fast": True},
                              {"name": "f", "type": "u64", "fast": True}]}


def _hash(d, mul, mod):
    return (d.astype(np.uint64) * np.uint64(mul)) % np.uint64(mod)


class Corpus:
    """Arrays of one split: term frequencies of body:x / u / v / w (0 = absent), doc lengths, columns a and f."""

    def __init__(self, n, tf, lens, a, f, split_id):
        self.n, self.tf, self.lens, self.a, self.f = n, tf, lens, a, f
        b = S._Builder(n)
        L = ffi.img_lib()
        uniq, inv = np.unique(lens, return_inverse=True)
        fn = np.array([L.qwgpu_fieldnorm_to_id(int(x)) for x in uniq], dtype=np.uint8)[inv]
        body = b.add_field("body", ffi.FIELD_HAS_FREQS | ffi.FIELD_HAS_FIELDNORMS, ffi.TOK_DEFAULT, fn, int(lens.sum()))
        for name in sorted(tf):
            docs = np.flatnonzero(tf[name]).astype(np.uint32)
            b.add_term(body, name.encode(), docs, tf[name][docs].astype(np.uint32))
        b.add_column("a", ffi.COL_U64, ffi.CARD_FULL, a.astype(np.uint64), None)
        b.add_column("f", ffi.COL_U64, ffi.CARD_FULL, f.astype(np.uint64), None)
        self.img = b.finish(split_id)
        self.norm = bm25_norm(lens)

    def under_id(self, split_id):
        """The same split registered under another id (another position in a batch)."""
        c = Corpus.__new__(Corpus)
        c.__dict__.update(self.__dict__)
        c.img = S.SplitImage(self.img.array, split_id)
        return c

    def scores(self, terms):
        """Union of `terms` in clause order: the numpy float32 restatement, with each term's weight checked against
        the compiled one (the plan carries the library's f32 idf; logf may differ from numpy's in the last place)."""
        s = np.zeros(self.n, dtype=np.float32)
        for t in terms:
            df = int(np.count_nonzero(self.tf[t]))
            w = np.float32(P.bm25_weight(df, self.n))
            assert abs(float(w) - float(bm25_weight(df, self.n))) <= 1e-6 * float(w)
            s = (s + bm25_contributions(self.tf[t], self.norm, w)).astype(np.float32)
        return s


def _benign(n, split_id):
    d = np.arange(n, dtype=np.int64)
    present = (d % 16) != 15
    tf = {"x": 1 + (d * 13) % 15,
          "u": np.where(present, 1 + (d * 7) % 15, 0), "v": np.where(present, 1, 0), "w": np.where(present, 1 + (d * 11) % 15, 0)}
    lens = 1 + _hash(d, 7919, 400).astype(np.int64)
    return Corpus(n, tf, lens, _hash(d, 2654435761, 1 << 32), d % 10, split_id)


def _h(K, s):
    """Top keys to put in one sampled window so that the sample alone reaches its target rank
    (k_pick: (2K + s - 1) / s + 24 unweighted, 2K + 24 s with the window weighted by s) while the split holds fewer
    than K docs at or above the threshold. Needs s >= 3."""
    return -(-2 * K // s) + 24 + 16


def _adversarial(n, W, s, scenario, K, split_id):
    """scenario "high": class 3 = _h(K, s) docs at the start of window s (sampled by every kernel at batch position
    0, with weight s under k_window), class 2 = every doc of windows 1..s-1 (never sampled: not strided, not an edge),
    class 1 = the rest. scenario "low": class 3 = TIE docs with one and the same top key, all but two in windows no
    sample reads. The classes order every sort of the module: column a DESC, score DESC over u (and x), score ASC
    over w."""
    d = np.arange(n, dtype=np.int64)
    win = d // W
    nw = (n + W - 1) // W
    cls = np.ones(n, dtype=np.int64)
    if scenario == "high":
        assert 3 <= s and s + 1 < nw and _h(K, s) < K and _h(K, s) <= W
        cls[(win >= 1) & (win < s)] = 2
        cls[s * W: s * W + _h(K, s)] = 3
    else:
        unsampled = np.flatnonzero((win % s != 0) & (win != 0) & (win != nw - 1))
        cls[unsampled[np.linspace(0, len(unsampled) - 1, TIE - 2).astype(np.int64)]] = 3
        cls[[s * W + 1, s * W + 5]] = 3
    present = ((d % 16) != 15) | (cls > 1)
    up = np.array([0, 1, 2, 15])[cls]            # score DESC: class 3 best
    down = np.array([0, 15, 2, 1])[cls]          # score ASC: class 3 best
    tf = {"x": up, "u": np.where(present, up, 0), "v": np.where(present, 1, 0), "w": np.where(present, down, 0)}
    lens = np.where((cls == 3) & (scenario == "low"), 10, 8 + d % 5)   # the tie shares its fieldnorm: one score
    r = _hash(d, 2654435761, 1 << 20).astype(np.int64)
    a = np.where(cls == 3, (0xFFFFFFFF if scenario == "low" else 0xC0000000 + r), np.where(cls == 2, 0x40000000 + r, r))
    f = np.where(cls > 1, 0, d % 10)
    return Corpus(n, tf, lens, a, f, split_id)


# ---- the sorts under test: (query, sort, kernel bit, brute force) ---------------------------------------------------
SCORE_ASC = [(ffi.SORT_SCORE, ffi.ORDER_ASC, ffi.ABSENT)]
CASES = ["union", "union_two_keys", "window_col", "window_score_asc", "driver_col", "driver_score"]
KERNEL = {"union": ffi.KERNEL_UNION, "union_two_keys": ffi.KERNEL_UNION, "window_col": ffi.KERNEL_WINDOW,
          "window_score_asc": ffi.KERNEL_WINDOW, "driver_col": ffi.KERNEL_DRIVER, "driver_score": ffi.KERNEL_DRIVER}


def _should(img, *terms):
    return P.bool_([P.term(img, "body", t, occur=ffi.OCCUR_SHOULD) for t in terms])


def _driver_root(img):
    return P.bool_([P.term(img, "body", "x", occur=ffi.OCCUR_MUST), P.range_(img, "f", 0, 8, occur=ffi.OCCUR_FILTER)])


def _plan(case, c, K, search_after=None):
    img = c.img
    root, sort = {
        "union": (_should(img, "u", "v"), SCORE_DESC),
        "union_two_keys": (_should(img, "u", "v"), [(ffi.SORT_SCORE, ffi.ORDER_DESC, ffi.ABSENT), col_sort(img, "a", ffi.ORDER_ASC)]),
        "window_col": (P.match_all(), [col_sort(img, "a", ffi.ORDER_DESC)]),
        "window_score_asc": (_should(img, "w", "v"), SCORE_ASC),
        "driver_col": (_driver_root(img), [col_sort(img, "a", ffi.ORDER_DESC)]),
        "driver_score": (_driver_root(img), SCORE_DESC),
    }[case]
    return P.make_plan(root, K, sort, search_after=search_after)


def _expected(case, c):
    """(matched docs in the sort's order, per-doc scores or None)."""
    d = np.arange(c.n, dtype=np.int64)
    a = c.a.astype(np.int64)
    if case in ("union", "union_two_keys"):
        m = (c.tf["u"] > 0) | (c.tf["v"] > 0)
        sc = c.scores(["u", "v"])
        keys = (-d, a, -sc) if case == "union_two_keys" else (-d, -sc)
    elif case == "window_score_asc":
        m = (c.tf["w"] > 0) | (c.tf["v"] > 0)
        sc = c.scores(["w", "v"])
        keys = (d, sc)
    elif case == "window_col":
        m, sc, keys = np.ones(c.n, dtype=bool), None, (-d, -a)
    else:
        m = (c.tf["x"] > 0) & (c.f <= 8)
        sc = c.scores(["x"]) if case == "driver_score" else None
        keys = (-d, -sc) if case == "driver_score" else (-d, -a)
    docs = d[m]
    order = np.lexsort(tuple(k[m] for k in keys))
    return docs[order], sc


def _check_brute(case, c, got, expected, K, ctx):
    order, sc = expected
    want = order[:K]
    assert [h[0] for h in got.hits] == want.tolist(), f"{ctx}: doc ids differ from the brute force"
    if sc is None:
        assert [h[2] for h in got.hits] == c.a[want].astype(np.int64).tolist(), f"{ctx}: sort values differ"
    else:
        gs = np.array([h[4] for h in got.hits], dtype=np.float32).view(np.uint32)
        assert np.array_equal(gs, sc[want].view(np.uint32)), f"{ctx}: f32 score bits differ from the restatement"
        if case == "union_two_keys":
            assert [h[3] for h in got.hits] == c.a[want].astype(np.int64).tolist(), f"{ctx}: second sort values differ"


def _path(r):
    return (f"kernel_mask={r.kernel_mask:#x} window_docs={r.window_docs} sample_stride={r.sample_stride} "
            f"exact_fallbacks={r.exact_fallbacks} refined={r.refined} radix_passes={r.radix_passes}")


def _run(ctx, case, corpora, K, label, search_after=None):
    """One batched call over `corpora`; every split checked against the oracle and the brute force."""
    plans = [_plan(case, c, K, search_after) for c in corpora]
    res = ctx.split_search([c.img.split_id for c in corpora], plans)
    print(f"[topk] {label} {case} K={K}: {_path(res[0])}")
    for i, (c, r, pl) in enumerate(zip(corpora, res, plans)):
        tag = f"{label} {case} K={K} split {i}"
        assert r.kernel_mask & KERNEL[case], f"{tag}: {_path(r)}"
        assert_same(r, O.split_search(c.img, pl), ctx=tag)
        if search_after is None:
            _check_brute(case, c, r, _expected(case, c), K, tag)
            assert r.num_hits == len(_expected(case, c)[0])
    return res[0]


# ---- corpora (built once per module) ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def benign(gpu_ctx):
    c = _benign(N, "topk-benign")
    gpu_ctx.register_split(c.img)
    yield c
    gpu_ctx.unregister_split(c.img.split_id)


@pytest.fixture(scope="module")
def probe(gpu_ctx, benign):
    """(window_docs, sample_stride) of every case on a 1 M-doc split, read back from the engine: k_window halves its
    window when shared memory does not fit, so the window size is not hard-coded here."""
    out = {}
    for case in CASES:
        r = gpu_ctx.split_search([benign.img.split_id], [_plan(case, benign, 10)])[0]
        assert r.sample_stride >= 3, f"{case}: {_path(r)}"
        out[case] = (r.window_docs, r.sample_stride)
    return out


_BUILT = {}


def _corpus(ctx, case, probe, scenario, K):
    W, s = probe[case]
    key = (W, s, scenario, K)
    if key not in _BUILT:
        _BUILT[key] = _adversarial(N, W, s, scenario, K, f"topk-{scenario}-{W}-{s}-{K}")
    c = _BUILT[key]
    if not ctx.is_resident(c.img.split_id):
        ctx.register_split(c.img)
    return c


@pytest.fixture(scope="module", autouse=True)
def _release(gpu_ctx):
    yield
    for c in _BUILT.values():
        if gpu_ctx.is_resident(c.img.split_id):
            gpu_ctx.unregister_split(c.img.split_id)
    _BUILT.clear()


# ---- tests ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES)
def test_sample_passes(gpu_ctx, benign, probe, case):
    """Benign keys: the sampled threshold holds; K = 1 and K = 4096 (max_hits + start_offset at its cap) included."""
    for K in (1, 100, 1000, 4096):
        r = _run(gpu_ctx, case, [benign], K, "passes")
        assert r.sample_stride >= 3
        if K <= 1000:  # (at K = 4096 the sample's own target is about the candidate capacity)
            assert r.exact_fallbacks == 0 and r.refined == 0 and r.radix_passes == 0, _path(r)


@pytest.mark.parametrize("case", CASES)
def test_sample_too_high(gpu_ctx, probe, case):
    """Too few candidates: column sorts with the level-0 histogram on record take the candidates-only repair; `_score`
    sorts and the posting-driven kernel re-run the exact radix descent."""
    K = 300
    c = _corpus(gpu_ctx, case, probe, "high", K)
    r = _run(gpu_ctx, case, [c], K, "too-high")
    assert r.sample_stride >= 3 and r.exact_fallbacks == 1 and r.radix_passes >= 1, _path(r)
    assert r.refined == (1 if case == "window_col" else 0), _path(r)
    W, s = probe[case]
    assert 1 <= r.hits[K - 1][0] // W < s, "the K-th hit lies in a window the sample never read"


@pytest.mark.parametrize("case", CASES)
def test_sample_too_low(gpu_ctx, probe, case):
    """More than QW_CAND_CAP docs share the top key: the collect pass overflows the candidate capacity and the exact
    descent resolves the tie down to the doc id."""
    for K in (1, 10):
        c = _corpus(gpu_ctx, case, probe, "low", 10)
        r = _run(gpu_ctx, case, [c], K, "too-low")
        assert r.sample_stride >= 3 and r.exact_fallbacks == 1 and r.radix_passes >= 1, _path(r)
        assert r.refined == (1 if case == "window_col" else 0), _path(r)


@pytest.mark.parametrize("case", ["union", "window_col"])
def test_mixed_batch(gpu_ctx, benign, probe, case):
    """One call: a 1 M-doc split that fails its sample (batch position 0), two that pass, and a small split with
    fewer windows than its sample phase (k_union reads none of its windows). The candidates of the passing splits
    must survive the repair of the failing one."""
    K = 300
    bad = _corpus(gpu_ctx, case, probe, "high", K)
    small = _benign(20_000, "topk-small")
    gpu_ctx.register_split(small.img)
    twin_c = benign.under_id("topk-benign-twin")
    gpu_ctx.register_split(twin_c.img)
    try:
        r = _run(gpu_ctx, case, [bad, benign, twin_c, small], K, "mixed")
        assert r.sample_stride >= 3 and r.exact_fallbacks == 1, _path(r)
        if case == "window_col":
            assert r.refined == 1, _path(r)
        # the same splits through qwgpu_leaf_search: per-split top-K merged on the device (k_merge_prep / k_merge)
        imgs = [bad.img, benign.img, twin_c.img, small.img]
        sort_fields = [("_score", proto.DESC)] if case == "union" else [("a", proto.DESC)]
        ast = bool_(should=[term("body", "u"), term("body", "v")]) if case == "union" else {"type": "match_all"}
        kw = dict(max_hits=K, sort_fields=sort_fields)
        offsets = [proto.enc_split_offsets(im.split_id, im.num_docs) for im in imgs]
        lreq = proto.enc_leaf_search_request(search_request(ast, **leafify(kw)), offsets, json.dumps(MAPPING))
        got = proto.dec_leaf_search_response(service.merge_leaf_responses(search_request(ast, **kw), [gpu_ctx.leaf_search(lreq)]))
        want = cpu_root_search(imgs, ast, MAPPING, **kw)
        assert got["num_hits"] == want["num_hits"] and got["partial_hits"] == want["partial_hits"]
    finally:
        gpu_ctx.unregister_split(small.img.split_id)
        gpu_ctx.unregister_split(twin_c.img.split_id)


@pytest.mark.parametrize("case", ["window_col", "driver_col"])
def test_search_after_with_a_failing_sample(gpu_ctx, probe, case):
    """search_after removes docs before the marker from the eligible count that the check compares against."""
    K = 300
    c = _corpus(gpu_ctx, case, probe, "high", K)
    order, _ = _expected(case, c)
    for rank in (5, 1000):
        marker = int(order[rank])
        sa = ffi.QwSearchAfter(1, 1, 0, 1, 0, marker, int(c.a[marker]), 0)
        r = _run(gpu_ctx, case, [c], K, f"search_after@{rank}", search_after=sa)
        assert r.sample_stride >= 3, _path(r)
        assert [h[0] for h in r.hits] == order[rank + 1: rank + 1 + K].tolist()
        assert r.num_hits == len(order)


# ---- k_select capacity edges -------------------------------------------------------------------------------------------
GROUPS = (2047, 2048, 2049, 8191, 8192, 8193)


def _tie_split(n, split_id):
    """Two 60-bit sort columns (the doc id falls outside the first key word). Column g<size> holds its maximum on
    `size` docs spread over the whole split; every other doc is far below. Column b orders within the tie with many
    equal values, so the doc id decides among those."""
    d = np.arange(n, dtype=np.int64)
    b = S._Builder(n)
    fid = b.add_field("body", ffi.FIELD_HAS_FREQS | ffi.FIELD_HAS_FIELDNORMS, ffi.TOK_DEFAULT, np.full(n, 1, np.uint8), n)
    b.add_term(fid, b"x", np.arange(n, dtype=np.uint32), np.ones(n, dtype=np.uint32))
    cols = {}
    top = (1 << 60) - 1
    for g in GROUPS:
        v = _hash(d, 2654435761 + g, 1 << 40)
        v[np.linspace(3, n - 1, g).astype(np.int64)] = top
        v[1] = 0
        cols[f"g{g}"] = v
        b.add_column(f"g{g}", ffi.COL_U64, ffi.CARD_FULL, v, None)
    bb = (d % 7).astype(np.uint64)
    bb[0] = top
    cols["b"] = bb
    b.add_column("b", ffi.COL_U64, ffi.CARD_FULL, bb, None)
    return b.finish(split_id), cols


@pytest.fixture(scope="module")
def tie_splits(gpu_ctx):
    out = {}
    for name, n in (("exact", 200_000), ("sampled", N)):
        img, cols = _tie_split(n, f"topk-ties-{name}")
        gpu_ctx.register_split(img)
        out[name] = (img, cols, n)
    yield out
    for img, _, _ in out.values():
        gpu_ctx.unregister_split(img.split_id)


@pytest.mark.parametrize("path", ["exact", "sampled"])
@pytest.mark.parametrize("g", GROUPS)
def test_select_capacity_edges(gpu_ctx, tie_splits, path, g):
    """Tie groups in the first 64-bit key word around QW_SEL_MAX (2048 survivors sorted in shared memory) and
    QW_CAND_CAP (8192 candidates); the K-th hit falls inside the tie."""
    img, cols, n = tie_splits[path]
    a, b = cols[f"g{g}"].astype(np.uint64), cols["b"].astype(np.uint64)
    d = np.arange(n, dtype=np.int64)
    order = np.lexsort((-d, b, ~a))           # g DESC, b ASC, doc id DESC (the direction of the first key)
    for K in (1000, min(g - 1, 4096)):
        pl = P.make_plan(P.match_all(), K, [col_sort(img, f"g{g}", ffi.ORDER_DESC), col_sort(img, "b", ffi.ORDER_ASC)])
        r = gpu_ctx.split_search([img.split_id], [pl])[0]
        print(f"[topk] ties {path} g={g} K={K}: {_path(r)}")
        assert r.kernel_mask & ffi.KERNEL_WINDOW
        assert (r.sample_stride >= 2) == (path == "sampled"), _path(r)
        if path == "exact":
            assert r.radix_passes >= 1
        assert_same(r, O.split_search(img, pl), ctx=f"ties {path} g={g} K={K}")
        want = order[:K]
        assert [h[0] for h in r.hits] == want.tolist()
        assert [h[2] for h in r.hits] == a[want].tolist() and [h[3] for h in r.hits] == b[want].tolist()
        if g > CAND_CAP and path == "sampled":
            assert r.exact_fallbacks == 1 and r.refined == 1, _path(r)
