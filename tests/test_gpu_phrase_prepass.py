"""The phrase, phrase-prefix and term-set pre-passes (k_phrase, k_phrase<true>, k_phrase_long, k_term_set) at their
limits (phrase_corpora.py), against phrase_ref's restatement from the arrays and against the oracle.

Every call's route is asserted from `kernel_mask`, and every result is compared bit for bit (doc ids, num_hits, f32
score bits) with the restatement and with the oracle (phrase prefixes and term sets rewritten for it):
  * each query of phrase_corpora.main_queries under `_score` desc at K = 1, 10, 1000, 4096, by doc id both ways, and
    count-only: driver and lookup shapes, repeated terms, offsets (gapped, above 0, not ascending; short, long and
    prefix), counts and fieldnorms, far positions, a position stream past 2^24, multi-valued gaps, phrase prefixes of
    1..7 exact terms and 1..1024 expansions, term sets on bitmap-word and round edges, the clauses inside bools;
  * phrase matches on the first doc of a window at every window size 2048..32768, scored and unscored, as MUST,
    SHOULD and FILTER, beside nested bools;
  * the offset docs "a b", "x a b", "b a" under offsets whose smallest is above 0 or that descend;
  * phrases of 2..8 terms alone and beside an 8-term phrase (the widest shared-memory layout);
  * a call of more than 200 phrases over several splits, and calls in sequence on one context (the call slot's
    pre-pass records, VBlk region and bitmaps reused);
  * refusals: 1025 expansions, 65 537 set terms, an offset spread of 2^31."""
import time

import numpy as np
import pytest

from quickwit_b200 import ffi, plan as P
from oracle import oracle as O
from helpers import assert_same
from phrase_prefix_ref import rewrite_as_phrases
from regex_ref import rewrite_term_sets
import phrase_corpora as PC
import phrase_ref as Q

pytestmark = pytest.mark.gpu

PHRASE, LONG, TERM_SET, WINDOW = ffi.KERNEL_PHRASE, ffi.KERNEL_PHRASE_LONG, ffi.KERNEL_TERM_SET, ffi.KERNEL_WINDOW
MAX_SET_TERMS = 65_536  # QW_MAX_SET_TERMS


@pytest.fixture(scope="module")
def main(gpu_ctx):
    t = time.time()
    c = PC.main_split()
    print(f"[phrase pre-pass] main split built in {time.time() - t:.1f} s")
    gpu_ctx.register_split(c.img)
    yield c
    gpu_ctx.unregister_split(c.img.split_id)


@pytest.fixture(scope="module")
def others(gpu_ctx):
    """The offset split, the 65 537-term split and six small splits."""
    cs = [PC.offset_split(), PC.many_terms_split()] + [PC.small_split(s) for s in range(6)]
    for c in cs:
        gpu_ctx.register_split(c.img)
    yield cs
    for c in cs:
        gpu_ctx.unregister_split(c.img.split_id)


def route(q):
    """The pre-pass bits a query's call must show."""
    m = WINDOW
    for cl in q.clauses:
        if cl.kind == "phrase":
            m |= PHRASE if len(cl.terms) <= ffi.MAX_PHRASE_TERMS else LONG
        elif cl.kind == "prefix":
            m |= PHRASE
        elif cl.kind == "term_set":
            m |= TERM_SET
    return m


PRE_PASSES = PHRASE | LONG | TERM_SET


def run(ctx, items, batch=64, oracle=True, exact=True):
    """items: (corpus, label, query, sort, K), every result checked. `kernel_mask` is call-wide, so with `exact` the
    items are grouped by route and each call's pre-pass bits must equal its plans' route (a short phrase sent to
    k_phrase_long shows); otherwise `batch` items go per call in order and the call must show every route of them."""
    out = []
    groups = {}
    for it in items:
        groups.setdefault(route(it[2]) if exact else 0, []).append(it)
    for key, its in groups.items():
        for i in range(0, len(its), batch):
            part = its[i:i + batch]
            plans = [q.plan(c.img, K, sort) for c, _, q, sort, K in part]
            got = ctx.split_search([c.img.split_id for c, *_ in part], plans)
            want = 0
            for _, _, q, _, _ in part:
                want |= route(q)
            for (c, label, q, sort, K), r, pl in zip(part, got, plans):
                tag = f"{label} {sort} K={K} kernel_mask={r.kernel_mask:#x}"
                assert r.kernel_mask & want == want, tag
                if exact:
                    assert r.kernel_mask & PRE_PASSES == want & PRE_PASSES, tag
                Q.check(r, c, q, K, sort, ctx=tag)
                if oracle:
                    assert_same(r, O.split_search(c.img, rewrite_as_phrases(rewrite_term_sets(pl))), ctx=tag)
            out += got
    return out


def test_main_queries(gpu_ctx, main):
    items = [(main, label, q, sort, K) for label, q in PC.main_queries() for sort, K in PC.sorts_for(q)]
    run(gpu_ctx, items)


def test_window_edges(gpu_ctx, main):
    """Phrase matches on the first doc of a window, at every window size 2048..32768, under driver blocks that
    straddle the edge: k_window folds such a block into the window before the edge too, where the doc lies one past
    the window's end and must be skipped. Each plan runs alone, so `window_docs` is its own."""
    seen = set()
    first, last = PC.block_bounds(main, "wedge", "we")
    for label, q in PC.edge_queries():
        for sort, K in (("score_desc", 4096), ("score_desc", 10), ("doc_asc", 4096), ("doc_desc", 0)):
            (r,) = run(gpu_ctx, [(main, label, q, sort, K)])
            w = r.window_docs
            seen.add(w)
            edges = np.arange(w, main.n, w)
            assert len(edges) and all(((first < e) & (e <= last)).any() for e in edges), (label, w)
    assert seen == set(PC.WINDOWS), sorted(seen)


def test_offsets_match_by_alignment(gpu_ctx, others):
    """Offsets (1, 2) and (5, 6) over "a b" match docs 0 and 1, (2, 1) doc 2: the smallest offset is not a start."""
    c = others[0]
    for offs, want in PC.offset_cases():
        q = Q.Query([Q.Phrase("body", ["a", "b"], offs)], bare=True)
        for sort, K in (("score_desc", 10), ("doc_asc", 10)):
            pl = q.plan(c.img, K, sort)
            r = gpu_ctx.split_search([c.img.split_id], [pl])[0]
            tag = f"offsets {offs} {sort}"
            assert r.kernel_mask & PHRASE, tag
            assert sorted(h[0] for h in r.hits) == want, tag
            Q.check(r, c, q, K, sort, ctx=tag)
            assert_same(r, O.split_search(c.img, pl), ctx=tag)
        # a phrase prefix over the same docs, the expansion `b`
        q = Q.Query([Q.Prefix("body", ["a"], ["b"], [offs[0]], offs[1], occur=Q.FILTER)])
        r = gpu_ctx.split_search([c.img.split_id], [q.plan(c.img, 10, "doc_asc")])[0]
        assert [h[0] for h in r.hits] == want, f"prefix offsets {offs}"


def test_layouts(gpu_ctx, main):
    """Phrases of 2..8 terms alone, then each in one call with an 8-term phrase: k_phrase sizes its shared memory
    by the longest phrase of the call."""
    eight = Q.Query([Q.Phrase("seq", PC.SEQ[:8], list(range(3, 11)))], bare=True)
    for k in range(2, 9):
        q = Q.Query([Q.Phrase("seq", PC.SEQ[:k], list(range(1, k + 1)))], bare=True)
        run(gpu_ctx, [(main, f"layout {k}", q, "score_desc", 1000)])
        run(gpu_ctx, [(main, f"layout {k} with 8", q, "score_desc", 1000), (main, "layout 8", eight, "doc_desc", 100)])


def _small_queries(c, seed):
    rng = np.random.default_rng(seed)
    vocab = ["a", "b"] + [f"v{i}" for i in range(10)]
    have = [t for t in vocab if ("body", t) in c.postings]
    qs = []
    for _ in range(26):
        k = int(rng.integers(2, 12))
        terms = [str(x) for x in rng.choice(have, k)]
        offs = (np.arange(k) + int(rng.integers(0, 4))).tolist()
        qs.append((f"small {terms}", Q.Query([Q.Phrase("body", terms, offs)], bare=True)))
    qs.append(("small a b x6", Q.Query([Q.Phrase("body", ["a", "b"] * 6)], bare=True)))
    exps = sorted(t for t in have if t.startswith("v"))
    qs.append(("small prefix", Q.Query([Q.Prefix("body", ["a", "b"], exps, occur=Q.FILTER)])))
    qs.append(("small prefix offsets", Q.Query([Q.Prefix("body", ["b"], exps[:3], [4], 5, occur=Q.FILTER)])))
    tsf = sorted(t for (f, t) in c.postings if f == "tsf")
    qs.append(("small term set", Q.Query([Q.TermSet("tsf", tsf[::3])])))
    return qs


def test_batch_of_200_phrases(gpu_ctx, main, others):
    """More than 200 pre-pass plans in one call over seven splits: the kernels' linear walk to their phrase runs
    long, and short, long and prefix phrases and term sets are numbered together."""
    items = [(main, label, q, "doc_desc", 100) for label, q in PC.main_queries()]
    for s, c in enumerate(others[2:]):
        items += [(c, label, q, "doc_desc", 100) for label, q in _small_queries(c, s)]
    assert sum(1 for _, _, q, _, _ in items if q.clauses[0].kind == "phrase") >= 200
    run(gpu_ctx, items, batch=len(items), exact=False)


def test_slot_reuse(gpu_ctx, main, others):
    """Calls in sequence on one context get the same call slot back: its pre-pass record arrays, VBlk region and
    term-set bitmaps must hold nothing of the call before."""
    smalls = others[2:]
    large = [(main, label, q, "doc_asc", 1000) for label, q in PC.main_queries()[::3]]
    for s, c in enumerate(smalls):
        large += [(c, label, q, "doc_asc", 1000) for label, q in _small_queries(c, 10 + s)[::2]]
    assert len({c.img.split_id for c, *_ in large}) >= 7
    one = [(main, "one phrase", Q.Query([Q.Phrase("body", ["ed", "lk"])], bare=True), "score_desc", 10)]
    ts_only = [(smalls[0], "term set only", Q.Query([Q.TermSet("tsf", sorted(t for (f, t) in smalls[0].postings if f == "tsf")[:5])]),
                "doc_desc", 4096)]
    nothing = [(main, "matches nothing", Q.Query([Q.Phrase("body", ["m1", "m2"], [0, 100])], bare=True), "doc_desc", 100)]
    for label, items in (("large", large), ("one", one), ("term set", ts_only), ("nothing", nothing), ("large again", large)):
        got = run(gpu_ctx, items, batch=len(items), exact=label in ("one", "term set", "nothing"))
        if label == "nothing":
            assert got[0].num_hits == 0 and got[0].hits == []


def test_many_terms(gpu_ctx, others):
    """A term set of 65 536 terms (the cap) is served; the restatement is the union of their doc lists."""
    c = others[1]
    terms = [f"k{j:05d}" for j in range(MAX_SET_TERMS)]
    q = Q.Query([Q.TermSet("k", terms)])
    for sort, K in (("doc_asc", 4096), ("doc_desc", 10), ("doc_desc", 0)):
        r = gpu_ctx.split_search([c.img.split_id], [q.plan(c.img, K, sort)])[0]
        assert r.kernel_mask & TERM_SET
        Q.check(r, c, q, K, sort, ctx=f"65536 terms {sort} K={K}")


def _code(ctx, c, node, sort="doc_asc"):
    with pytest.raises(ffi.QwGpuError) as e:
        ctx.split_search([c.img.split_id], [P.make_plan(node, 10, Q.SORTS[sort])])
    return e.value.code


def test_refusals(gpu_ctx, main, others):
    many = others[1]
    img = main.img
    # 1025 expansions
    node = Q.Prefix("seq", ["s00"], PC._expansions(1025), occur=Q.FILTER).node(img)
    assert _code(gpu_ctx, main, P.bool_([node])) == ffi.EUNSUPPORTED
    # 65 537 set terms
    node = Q.TermSet("k", [f"k{j:05d}" for j in range(PC.MANY_TERMS)]).node(many.img)
    assert len(node.children) == PC.MANY_TERMS
    assert _code(gpu_ctx, many, P.bool_([node])) == ffi.EINVALID_ARG
    # an offset spread of 2^31 (short, long, prefix); 2^31 - 1 is served
    big = 1 << 31
    for ph in (Q.Phrase("far", ["fa", "fb"], [0, big]), Q.Phrase("far", ["fb", "fa"], [big + 5, 5]),
               Q.Phrase("seq", PC.SEQ[:9], list(range(8)) + [big])):
        assert _code(gpu_ctx, main, ph.node(img)) == ffi.EINVALID_ARG, ph.label()
    px = Q.Prefix("seq", ["s00"], ["s01"], [0], big, occur=Q.FILTER)
    assert _code(gpu_ctx, main, P.bool_([px.node(img)])) == ffi.EINVALID_ARG
    ok = Q.Query([Q.Phrase("far", ["fa", "fb"], [0, big - 1])], bare=True)
    run(gpu_ctx, [(main, "spread 2^31 - 1", ok, "doc_asc", 10)])
