"""k_select, the final top-K of every split with K <= 4096, against a brute-force sort of the same documents' keys.

k_select cuts each split's candidates to the survivors whose first key word reaches the K-th largest one, then ranks
every survivor by counting the larger keys of its rank bucket and the buckets above (QW_SEL_TILES blocks per split,
buckets picked by the key bits after those all survivors share); a split with more than
QW_SEL_MAX = 2048 survivors (ties on the first key word) is sorted whole instead. Covered here on k_union, k_driver
and k_window (asserted through kernel_mask):
  * K = 1, 10, 1000, 4096 over splits matching K - 1, K, K + 1 and QW_CAND_CAP documents;
  * two-field column sorts whose top documents share the first key word (a 40-bit column, then the high bits of a
    second one), with QW_SEL_MAX and QW_SEL_MAX + 1 of them, in both directions;
  * splits asking for no hits in one batch with top-K splits;
  * the sampled k_union path on splits of 2^20 documents.
Every split is checked bit for bit against the oracle and its doc ids against numpy's lexsort of the sort values."""
import numpy as np
import pytest

from quickwit_b200 import ffi, plan as P, splitgen as S
from oracle import oracle as O
from helpers import SCORE_DESC, assert_same, bm25_contributions, bm25_norm, col_sort

pytestmark = pytest.mark.gpu

CAND_CAP = 8192      # QW_CAND_CAP
SEL_MAX = 2048       # QW_SEL_MAX
AMAX = (1 << 40) - 1  # column range: a two-field key is wider than one 64-bit word


def _hash(d, mul, mod):
    return (d.astype(np.uint64) * np.uint64(mul)) % np.uint64(mod)


class Corpus:
    """One split: body terms u, v (every doc), x (3 docs of 4); u64 columns a and f over [0, AMAX].
    `tie` docs (spread over the split) share a = tie_a and the high bits of f, so their keys tie on the first word."""

    def __init__(self, n, split_id, tie=0, tie_a=AMAX):
        d = np.arange(n, dtype=np.int64)
        a = _hash(d, 2654435761, AMAX - 1).astype(np.int64) + 1
        f = _hash(d, 40503, AMAX + 1).astype(np.int64)
        a[0], a[-1] = 0, AMAX
        if tie:
            t = np.linspace(2, n - 1, tie).astype(np.int64)
            a[1] = AMAX - tie_a  # the other end of the column range
            a[t] = tie_a
            f[t] = (1 << 39) + (t * 7) % 1000
        self.n, self.a, self.f = n, a, f
        self.tf = {"u": 1 + (d * 13) % 7, "v": np.ones(n, dtype=np.int64), "x": np.where(d % 4 != 3, 1 + d % 5, 0)}
        lens = 1 + _hash(d, 7919, 300).astype(np.int64)
        b = S._Builder(n)
        L = ffi.img_lib()
        uniq, inv = np.unique(lens, return_inverse=True)
        fn = np.array([L.qwgpu_fieldnorm_to_id(int(x)) for x in uniq], dtype=np.uint8)[inv]
        body = b.add_field("body", ffi.FIELD_HAS_FREQS | ffi.FIELD_HAS_FIELDNORMS, ffi.TOK_DEFAULT, fn, int(lens.sum()))
        for name in sorted(self.tf):
            docs = np.flatnonzero(self.tf[name]).astype(np.uint32)
            b.add_term(body, name.encode(), docs, self.tf[name][docs].astype(np.uint32))
        b.add_column("a", ffi.COL_U64, ffi.CARD_FULL, a.astype(np.uint64), None)
        b.add_column("f", ffi.COL_U64, ffi.CARD_FULL, f.astype(np.uint64), None)
        self.img = b.finish(split_id)
        self.norm = bm25_norm(lens)

    def scores(self, terms):
        s = np.zeros(self.n, dtype=np.float32)
        for t in terms:
            w = np.float32(P.bm25_weight(int(np.count_nonzero(self.tf[t])), self.n))
            s = (s + bm25_contributions(self.tf[t], self.norm, w)).astype(np.float32)
        return s


ROUTES = {"union": ffi.KERNEL_UNION, "driver": ffi.KERNEL_DRIVER, "window": ffi.KERNEL_WINDOW}


def _plan(route, c, K, sort=None):
    img = c.img
    if route == "union":
        root = P.bool_([P.term(img, "body", t, occur=ffi.OCCUR_SHOULD) for t in ("u", "v")])
        return P.make_plan(root, K, sort or SCORE_DESC)
    if route == "driver":
        root = P.bool_([P.term(img, "body", "x", occur=ffi.OCCUR_MUST), P.range_(img, "f", 0, AMAX, occur=ffi.OCCUR_FILTER)])
        return P.make_plan(root, K, sort or [col_sort(img, "a", ffi.ORDER_DESC)])
    return P.make_plan(P.match_all(), K, sort or [col_sort(img, "a", ffi.ORDER_DESC)])


def _brute(route, c, fields):
    """Doc ids of the split's matches in the order of `fields` [(name, desc)], doc id last in the first one's
    direction."""
    d = np.arange(c.n, dtype=np.int64)
    m = c.tf["x"] > 0 if route == "driver" else np.ones(c.n, dtype=bool)
    vals = {"a": c.a, "f": c.f}
    if any(name == "_score" for name, _ in fields):
        vals["_score"] = c.scores(["u", "v"]).astype(np.float64)
    keys = [d if not fields[0][1] else -d]
    for name, desc in reversed(fields):
        keys.append(-vals[name] if desc else vals[name])
    return d[m][np.lexsort(tuple(k[m] for k in keys))]


def _path(r):
    return f"kernel_mask={r.kernel_mask:#x} sample_stride={r.sample_stride} exact_fallbacks={r.exact_fallbacks}"


def _check(ctx, corpora, Ks, route, fields, label, sort=None, kernel=True):
    plans = [_plan(route, c, K, sort) for c, K in zip(corpora, Ks)]
    res = ctx.split_search([c.img.split_id for c in corpora], plans)
    for i, (c, r, pl, K) in enumerate(zip(corpora, res, plans, Ks)):
        tag = f"{label} split {i} ({_path(r)})"
        assert not kernel or r.kernel_mask & ROUTES[route], tag
        assert_same(r, O.split_search(c.img, pl), ctx=tag)
        want = _brute(route, c, fields)[:K]
        assert [h[0] for h in r.hits] == list(want), f"{tag}: doc ids differ from the brute force"
    return res


@pytest.fixture(scope="module")
def registered(gpu_ctx):
    ids = []

    def reg(c):
        gpu_ctx.register_split(c.img)
        ids.append(c.img.split_id)
        return c
    yield reg
    for i in ids:
        gpu_ctx.unregister_split(i)


@pytest.mark.parametrize("route", sorted(ROUTES))
@pytest.mark.parametrize("K", [1, 10, 1000, 4096])
def test_select_counts(gpu_ctx, registered, route, K):
    """Splits matching K - 1, K, K + 1 and QW_CAND_CAP docs in one batch."""
    # docs per split so that m of them match (k_driver's query matches docs 0, 1, 2 of every 4)
    sizes = sorted({m + m // 3 if route == "driver" else m for m in (K - 1, K, K + 1, CAND_CAP) if m > 0})
    corpora = [registered(Corpus(n, f"sel-{route}-{K}-{n}")) for n in sizes]
    fields = [("_score", True)] if route == "union" else [("a", True)]
    _check(gpu_ctx, corpora, [K] * len(corpora), route, fields, f"{route} K={K}")


@pytest.mark.parametrize("tie", [SEL_MAX, SEL_MAX + 1])
@pytest.mark.parametrize("dirs", [(True, False), (False, True)])
@pytest.mark.parametrize("route", ["window", "driver"])
def test_select_first_word_ties(gpu_ctx, registered, route, dirs, tie):
    """QW_SEL_MAX (ranked) and QW_SEL_MAX + 1 (sorted whole) top docs tied on the first key word, K = 1000."""
    da, df = dirs
    c = registered(Corpus(20_000, f"sel-tie-{route}-{int(da)}{int(df)}-{tie}", tie=tie, tie_a=AMAX if da else 0))
    sort = [col_sort(c.img, "a", ffi.ORDER_DESC if da else ffi.ORDER_ASC), col_sort(c.img, "f", ffi.ORDER_DESC if df else ffi.ORDER_ASC)]
    _check(gpu_ctx, [c], [1000], route, [("a", da), ("f", df)], f"{route} tie={tie} dirs={dirs}", sort)


def test_select_union_two_keys_ties(gpu_ctx, registered):
    """_score DESC then a ASC on k_union: docs with the same tf and length tie on the score."""
    c = registered(Corpus(20_000, "sel-union-two"))
    sort = [(ffi.SORT_SCORE, ffi.ORDER_DESC, ffi.ABSENT), col_sort(c.img, "a", ffi.ORDER_ASC)]
    _check(gpu_ctx, [c], [1000], "union", [("_score", True), ("a", False)], "union two keys", sort)


@pytest.mark.parametrize("route", sorted(ROUTES))
def test_select_no_hit_splits_in_batch(gpu_ctx, registered, route):
    """Count-only splits (max_hits = 0) between top-K splits; such a batch may leave the route's own kernel."""
    corpora = [registered(Corpus(5000 + 37 * i, f"sel-zero-{route}-{i}")) for i in range(4)]
    fields = [("_score", True)] if route == "union" else [("a", True)]
    res = _check(gpu_ctx, corpora, [1000, 0, 1000, 0], route, fields, f"{route} zero-hit mix", kernel=False)
    assert [len(r.hits) for r in res[1::2]] == [0, 0]


def test_select_sampled_union(gpu_ctx, registered):
    """Splits of 2^20 docs: k_union samples its threshold before collecting."""
    corpora = [registered(Corpus(1 << 20, f"sel-big-{i}")) for i in range(4)]
    res = _check(gpu_ctx, corpora, [1000] * 4, "union", [("_score", True)], "sampled union")
    print(f"[select] sampled union: {_path(res[0])}")
