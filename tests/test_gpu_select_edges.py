"""k_select at its edges, on k_window and k_driver (and `_score` on k_union), against the 192-bit brute force of
tests/select_ref.py and the oracle.

The cases (labelled on the host by tests/test_select_rank_host.py) put the rank path's bucket bits at every shared-prefix
length p (across the word-0/1 and word-1/2 boundaries, over both has-value bits, inside the doc-id bits), stop the cut at
each of its shifts with QW_SEL_MAX survivors and one more, take K and the match count across every edge (K above
QW_SEL_MAX on the rank path, 1..5 survivors over the four tiles), decode missing values, a 1-doc split and doc-id sorts,
and sort splits of n far from a power of two whole, one of them holding an all-zero key. Every call asserts its route
from kernel_mask and that no sampled threshold ran (sample_stride == 0), so the restated candidate set is the one
k_select saw. Each split is checked bit for bit against the oracle and its doc ids against the sorted keys."""
import numpy as np
import pytest

from quickwit_b200 import ffi
from oracle import oracle as O
from helpers import assert_same
import select_ref as R

pytestmark = pytest.mark.gpu

ROUTES = {"window": ffi.KERNEL_WINDOW, "driver": ffi.KERNEL_DRIVER}
BATCH = 8  # top-K splits per call (k_select's grid: 4 x splits, zero-hit splits included)
GROUPS = R.all_cases()


@pytest.fixture(scope="module")
def registered(gpu_ctx):
    imgs = []  # (kept alive while registered)

    def reg(img):
        gpu_ctx.register_split(img)
        imgs.append(img)
        return img
    yield reg
    for img in imgs:
        gpu_ctx.unregister_split(img.split_id)


@pytest.fixture(scope="module")
def zero_splits(registered):
    """Splits asked for no hits, placed between the top-K splits of every batch."""
    out = []
    for i in range(BATCH // 2):
        c = R.edge_cases()[i]
        out.append((c, {r: registered(c.image(f"sel-edge-zero-{r}-{i}")) for r in ROUTES}))
    return out


def _tag(r):
    return f"kernel_mask={r.kernel_mask:#x} sample_stride={r.sample_stride} radix_passes={r.radix_passes}"


def _run(ctx, registered, zero_splits, cases, route):
    for b in range(0, len(cases), BATCH):
        batch = cases[b:b + BATCH]
        entries = []  # (case, img, plan)
        for i, c in enumerate(batch):
            img = registered(c.image(f"sel-edge-{route}-{c.name}"))
            entries.append((c, img, c.plan(img, route)))
            if i % 2 == 1:
                zc, zimg = zero_splits[i // 2]
                entries.append((zc, zimg[route], zc.plan(zimg[route], route, K=0)))
        res = ctx.split_search([e[1].split_id for e in entries], [e[2] for e in entries])
        for (c, img, plan), r in zip(entries, res):
            zero = c not in batch
            tag = f"{route} {c.name}{' (no hits asked)' if zero else ''} ({_tag(r)}) {'' if zero else c.label()}"
            assert r.kernel_mask & ROUTES[route], tag
            assert r.sample_stride == 0, tag
            if zero:
                assert r.hits == [] and r.num_hits == len(c.matched), tag
                continue
            assert_same(r, O.split_search(img, plan), ctx=tag)
            want = c.layout().brute_docs(c.matched)[:c.K]
            assert [h[0] for h in r.hits] == want, f"{tag}: doc ids differ from the brute force"


@pytest.mark.parametrize("route", sorted(ROUTES))
@pytest.mark.parametrize("group", ["at", "cut", "edge", "decode", "pad"])
def test_select_edges(gpu_ctx, registered, zero_splits, group, route):
    _run(gpu_ctx, registered, zero_splits, GROUPS[group], route)


def test_select_score_union(gpu_ctx, registered):
    """`_score` alone (8-byte QwScoreHit records) and `_score, b ASC` (QwHit) plans in one k_union batch, K = 2047, 2048
    and 2049, over top score groups of 2048 and 2049 tied docs: the survivors land on both sides of QW_SEL_MAX."""
    cases = R.score_cases()
    imgs = [registered(sp.image(f"sel-edge-{name}")) for name, sp, _, _ in cases]
    plans = [sp.plan(img, K, wb) for img, (_, sp, K, wb) in zip(imgs, cases)]
    res = gpu_ctx.split_search([i.split_id for i in imgs], plans)
    for img, plan, (name, sp, K, wb), r in zip(imgs, plans, cases, res):
        lay = sp.layout(wb)
        tag = f"{name} ({_tag(r)}) {R.restate(lay.keys(range(sp.n)), K, lay.total_bits)}"
        assert r.kernel_mask & ffi.KERNEL_UNION, tag
        assert r.sample_stride == 0, tag
        assert_same(r, O.split_search(img, plan), ctx=tag)
        assert [h[0] for h in r.hits] == lay.brute_docs(range(sp.n))[:K], f"{tag}: doc ids differ from the brute force"
        got = np.array([h[4] for h in r.hits], dtype=np.float32).view(np.uint32)
        want = sp.scores()[[h[0] for h in r.hits]].view(np.uint32)
        assert np.array_equal(got, want), f"{tag}: scores differ from the float32 BM25 restatement"
