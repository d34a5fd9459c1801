"""Posting decode and BM25 scoring on every decoder, at every packed width, tf and fieldnorm id (posting_corpora.py).

Each call is routed through one decoder, and the route is asserted from `kernel_mask`:
  * k_union: pure ORs of up to 32 sweep terms under `_score` desc, K = 1, 100, 4096; the mixed-width warp steps;
    boosts other than 1; a batch of splits with their own BM25 tables (the sweep, a 1-doc split, the 2^24-doc split);
  * k_window: the same unions by `_score` ascending, with a `must` clause, and by doc id (unscored: no tfs read);
    a batch with an empty split and a split without the terms (plans k_union does not take);
  * k_driver: one term per call, scored, with and without a range filter;
  * k_phrase: the phrase pairs by `_score` and by doc id, and one phrase prefix over expansions of every width;
  * k_term_set: a term-set filter over the terms of each doc width, of the tf-width sweep and of each other field.
Every result is compared bit for bit with scoring_ref's f32 restatement and with the oracle, and within the f64
bound of scoring_ref.f64_bound."""
import time

import numpy as np

import pytest

from quickwit_b200 import ffi, plan as P
from oracle import oracle as O
from helpers import assert_same
from regex_ref import oracle_search
import posting_corpora as PC
import scoring_ref as R

pytestmark = pytest.mark.gpu

UNION, WINDOW, DRIVER, PHRASE = ffi.KERNEL_UNION, ffi.KERNEL_WINDOW, ffi.KERNEL_DRIVER, ffi.KERNEL_PHRASE
TERM_SET = ffi.KERNEL_TERM_SET


@pytest.fixture(scope="module")
def sweep(gpu_ctx):
    t = time.time()
    c = PC.sweep_split()
    print(f"[widths] sweep split built in {time.time() - t:.1f} s")
    gpu_ctx.register_split(c.img)
    yield c
    gpu_ctx.unregister_split(c.img.split_id)


@pytest.fixture(scope="module")
def others(gpu_ctx):
    """The 2^24-doc split, the 1-doc split and the empty split."""
    cs = (PC.large_split(), PC.tiny_split(), PC.empty_split())
    for c in cs:
        gpu_ctx.register_split(c.img)
    yield cs
    for c in cs:
        gpu_ctx.unregister_split(c.img.split_id)


def _run(ctx, c, clauses, K, sort="score_desc", must=None, filt=False, route=UNION, label=""):
    pl = R.plan(c, clauses, K, sort, must, filt)
    r = ctx.split_search([c.img.split_id], [pl])[0]
    tag = f"{label} {sort} K={K} kernel_mask={r.kernel_mask:#x} window_docs={r.window_docs}"
    assert r.kernel_mask & route, tag
    if route != UNION:
        assert not r.kernel_mask & UNION, tag
    assert_same(r, O.split_search(c.img, pl), ctx=tag)
    R.check(r, c, clauses, K, sort, must, filt, ctx=tag)
    return r


def test_union(gpu_ctx, sweep):
    groups = PC.union_groups(sweep)
    for gi, g in enumerate(groups):
        for K in (1, 100, 4096):
            r = _run(gpu_ctx, sweep, g, K, label=f"union group {gi}")
            assert r.window_docs == PC.UNION_W
    for gi in (0, len(groups) // 2, len(groups) - 2, len(groups) - 1):
        for K in (100, 4096):
            _run(gpu_ctx, sweep, PC.boosted(groups[gi]), K, label=f"union boosted group {gi}")


def test_union_mixed_width_warp_steps(gpu_ctx, sweep):
    """Single-block clauses in one window: a narrow block (doc and tf widths <= 16) paired in one warp step with a
    wide one, so the warp's `narrow` vote is false for the narrow block, in either order."""
    for g in PC.mixed_groups():
        for cl in g:
            assert len(sweep.intended[(cl.field, cl.terms[0])]) == 1
            assert PC.UNION_W <= sweep.postings[(cl.field, cl.terms[0])][0][0] < 2 * PC.UNION_W
        for K in (1, 100, 4096):
            _run(gpu_ctx, sweep, g, K, label=f"mixed {[cl.terms[0] for cl in g]}")
        _run(gpu_ctx, sweep, PC.boosted(g), 100, label=f"mixed boosted {[cl.terms[0] for cl in g]}")


def test_window(gpu_ctx, sweep):
    groups = PC.union_groups(sweep)
    dense = R.Clause("body", ["dense"])
    for gi, g in enumerate(groups):
        for K in (100, 4096):
            _run(gpu_ctx, sweep, g, K, "score_asc", route=WINDOW, label=f"window group {gi}")
        _run(gpu_ctx, sweep, g, 4096, "doc_desc", route=WINDOW, label=f"window unscored group {gi}")
        gm = g[:31] + [dense]
        _run(gpu_ctx, sweep, gm, 100, must=len(gm) - 1, route=WINDOW, label=f"window must group {gi}")
    for g in PC.mixed_groups()[:2]:
        _run(gpu_ctx, sweep, g, 100, "score_asc", route=WINDOW, label="window mixed")


def test_driver(gpu_ctx, sweep):
    for f, t in PC.driver_terms(sweep):
        for filt in (False, True):
            _run(gpu_ctx, sweep, [R.Clause(f, [t])], 100, must=0, filt=filt, route=DRIVER, label=f"driver {f}:{t} filt={filt}")


def test_phrase(gpu_ctx, sweep):
    for cl in PC.phrase_pairs(sweep):
        for sort in ("score_desc", "doc_desc"):
            _run(gpu_ctx, sweep, [cl], 4096, sort, must=0, route=PHRASE, label=f"phrase {cl.terms}")
    node = P.phrase_prefix(sweep.img, "ph", ["pa05_000", "pb"], 50)
    assert node.kind == ffi.NODE_PHRASE_PREFIX and len(node.children) - 1 == len(sweep.terms_of("ph", "pb"))
    r = gpu_ctx.split_search([sweep.img.split_id], [P.make_plan(node, 4096, R.SORTS["doc_desc"])])[0]
    assert r.kernel_mask & PHRASE
    want = R.phrase_prefix_docs(sweep, "ph", "pa05_000", "pb")
    assert len(want) > 0 and r.num_hits == len(want) and [h[0] for h in r.hits] == want[::-1].tolist()
    # (the oracle runs the same match set as an OR of one phrase per expansion)
    assert_same(r, O.split_search(sweep.img, P.make_plan(P.phrase_prefix_as_phrases(node), 4096, R.SORTS["doc_desc"])), ctx="phrase prefix")


def test_term_set(gpu_ctx, sweep):
    """A TERM_SET filter over each group's terms: its doc set is the union of the terms' postings, at most 16 517
    docs, so one page of K = 20 000 holds all of it."""
    img = sweep.img
    gpu_ctx.set_max_hits(20_000)
    try:
        for field, terms in PC.term_set_groups(sweep):
            want = np.unique(np.concatenate([sweep.postings[(field, t)][0] for t in terms]))
            assert 0 < len(want) <= 20_000
            node = P.bool_([P.term_set(img, field, sorted(img.term_ord(field, t) for t in terms))])
            for sort, docs in (("doc_desc", want[::-1]), ("doc_asc", want)):
                pl = P.make_plan(node, 20_000, R.SORTS[sort])
                r = gpu_ctx.split_search([img.split_id], [pl])[0]
                tag = f"term set {field}:{terms[0]}..{terms[-1]} ({len(terms)} terms) {sort} kernel_mask={r.kernel_mask:#x}"
                assert r.kernel_mask & TERM_SET and r.kernel_mask & WINDOW, tag
                assert r.num_hits == len(want) and [h[0] for h in r.hits] == docs.tolist(), tag
                assert_same(r, oracle_search(img, pl), ctx=tag)
    finally:
        gpu_ctx.set_max_hits(4096)


def test_large_split(gpu_ctx, others):
    large = others[0]
    for gi, g in enumerate(PC.union_groups(large)):
        for K in (1, 100, 4096):
            _run(gpu_ctx, large, g, K, label=f"large group {gi}")
        _run(gpu_ctx, large, g, 100, "score_asc", route=WINDOW, label=f"large window group {gi}")
        for cl in g:
            _run(gpu_ctx, large, [cl], 10, must=0, route=DRIVER, label=f"large driver {cl.terms[0]}")


def test_multi_split_batch(gpu_ctx, sweep, others):
    """One call over splits that each bring their own BM25 tables: the persistent grid changes plan mid-chunk. The
    k_union batch holds the sweep, the 1-doc split and the 2^24-doc split; a split without the terms, or an empty
    one, lowers to a plan k_union does not take, so those ride in a second batch, on k_window."""
    large, tiny, empty = others
    g_sweep, g_large, g_tiny = PC.union_groups(sweep)[3], PC.union_groups(large)[0], PC.union_groups(tiny)[0]
    for K in (1, 100, 4096):
        batch = [(sweep, g_sweep), (tiny, g_tiny), (large, g_large), (sweep, PC.union_groups(sweep)[-2])]
        plans = [R.plan(c, g, K) for c, g in batch]
        res = gpu_ctx.split_search([c.img.split_id for c, _ in batch], plans)
        for i, ((c, g), r, pl) in enumerate(zip(batch, res, plans)):
            tag = f"batch K={K} split {i} kernel_mask={r.kernel_mask:#x}"
            assert r.kernel_mask & UNION, tag
            assert_same(r, O.split_search(c.img, pl), ctx=tag)
            R.check(r, c, g, K, ctx=tag)
        absent = [R.Clause("body", ["tf05"]), R.Clause("body", ["w03_000"])]   # (tiny has w00_000 and w01_000 only)
        batch = [(sweep, g_sweep), (empty, absent), (tiny, absent), (large, g_large), (tiny, g_tiny)]
        plans = [R.plan(c, g, K) for c, g in batch]
        res = gpu_ctx.split_search([c.img.split_id for c, _ in batch], plans)
        for i, ((c, g), r, pl) in enumerate(zip(batch, res, plans)):
            tag = f"batch+absent K={K} split {i} kernel_mask={r.kernel_mask:#x}"
            assert r.kernel_mask & WINDOW and not r.kernel_mask & UNION, tag
            assert_same(r, O.split_search(c.img, pl), ctx=tag)
            if g is absent:
                assert r.num_hits == 0 and r.hits == [], tag
            else:
                R.check(r, c, g, K, ctx=tag)
