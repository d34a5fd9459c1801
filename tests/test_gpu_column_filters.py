"""Fast-field range / exists filters and column sort keys on every kernel, against column_ref's brute force (built
from the source arrays, never the image) and the oracle, bit for bit.

Routes, asserted from `kernel_mask` on every call:
  * k_driver (KERNEL_DRIVER, never KERNEL_WINDOW): term AND 1..4 range / exists filters over every column of the
    main split at every bound point (driver_cases); term-driven sorts and paging;
  * k_window scan: a range / exists as the only required clause, should with minimum_should_match, must_not, nested
    bools, scored range clauses under _score (scan_cases); range-driven sorts and paging;
  * k_window gather: term AND term AND range over the q128 / q129 / sparse / all candidate sets, and range AND range
    (gather_cases);
  * sort keys: every width as the first key (QW_TOP_COLUMN from 10 bits up, QW_TOP_FULL below), the key pairs of
    exactly 64 bits (narrow), 65 bits and three words (wide); doc-id sorts on the 1-doc split (QW_TOP_FULL), the
    1024-doc split (doc_bits 10: QW_TOP_FULL) and the 2048- and 2049-doc splits (doc_bits 11 and 12: QW_TOP_DOC);
  * the device merge of one leaf request over splits whose fields differ in width, min and gcd.
Each call batches several plans over the same split, so that a plan the compiler lowers to "matches nothing" (a
range wholly outside the column) still runs beside plans that launch the route's kernel."""
import math
import time

import pytest

from quickwit_b200 import ffi, splitgen as S
from quickwit_b200.proto import ASC, DESC
from oracle import oracle as O
from helpers import assert_same
from pipeline import cpu_root_search
from test_gpu_leaf_search import gpu_root_search
import column_corpora as CC
import column_ref as R
import test_column_filters_host as H

pytestmark = pytest.mark.gpu

DRIVER, WINDOW, UNION = ffi.KERNEL_DRIVER, ffi.KERNEL_WINDOW, ffi.KERNEL_UNION
BATCH = 8


@pytest.fixture(scope="module")
def main(gpu_ctx):
    t = time.time()
    sp = CC.main_split()
    print(f"[columns] main split built in {time.time() - t:.1f} s")
    gpu_ctx.register_split(sp.img)
    yield sp
    gpu_ctx.unregister_split(sp.split_id)


@pytest.fixture(scope="module")
def smalls(gpu_ctx):
    sps = [CC.small_split(n) for n in CC.SMALL_DOCS]
    for sp in sps:
        gpu_ctx.register_split(sp.img)
    yield sps
    for sp in sps:
        gpu_ctx.unregister_split(sp.split_id)


def _route_ok(r, route, tag):
    if route == DRIVER:
        assert r.kernel_mask & DRIVER and not r.kernel_mask & WINDOW, tag
    else:
        assert r.kernel_mask & WINDOW and not r.kernel_mask & (DRIVER | UNION), tag


def run(ctx, items, route, label="", batch=BATCH):
    """items: (split, Q, Sort, K, search_after, scored, aggs). One split_search call per `batch` items; every result is
    compared with the oracle and with the brute force. Returns the results."""
    out = []
    for i0 in range(0, len(items), batch):
        chunk = items[i0:i0 + batch]
        plans = [R.plan(sp, q, sort, K, sa, aggs) for sp, q, sort, K, sa, _, aggs in chunk]
        res = ctx.split_search([it[0].split_id for it in chunk], plans)
        for (sp, q, sort, K, sa, scored, aggs), r, pl in zip(chunk, res, plans):
            tag = f"{label} {sp.split_id} {q!r} sort={sort.keys} K={K} kernel_mask={r.kernel_mask:#x}"
            _route_ok(r, route, tag)
            assert_same(r, O.split_search(sp.img, pl), ctx=tag)
            R.check(r, sp, q, sort, K, sa, scored, ctx=tag)
            out.append(r)
    return out


def item(sp, q, sort, K, sa=None, scored=False, aggs=()):
    return (sp, q, sort, K, sa, scored, aggs)


def test_driver_filters_on_every_width_and_bound(gpu_ctx, main):
    cases = R.driver_cases(main)
    assert any("below" in c[0] for c in cases) and any("above" in c[0] for c in cases)
    run(gpu_ctx, [item(main, q, sort, K) for _, q, sort, K in cases], DRIVER, "driver")


def test_window_scan(gpu_ctx, main):
    run(gpu_ctx, [item(main, q, sort, K, scored=scored) for _, q, sort, K, scored in R.scan_cases(main)], WINDOW, "scan")


def test_window_gather(gpu_ctx, main):
    run(gpu_ctx, [item(main, q, sort, K) for _, q, sort, K in R.gather_cases(main)], WINDOW, "gather")
    # term AND range with an aggregation: the plan stays off k_driver, the range gathers over the term's docs
    stats = [R.P.Agg(ffi.AGG_STATS, column=main.ords["w20"])]
    items = []
    for t in R.GATHER_TERMS:
        for name in ("w33", "m64", "o9"):
            lo, hi = R._wide(main, name, None)
            items.append(item(main, R.bool_([R.term(t), R.rng(name, lo, hi)]), R.col_sort(name, ASC), 100, aggs=stats))
    run(gpu_ctx, items, WINDOW, "gather+agg")


def test_sort_keys_on_every_width(gpu_ctx, main):
    everything = R.bool_([R.rng("w0", 0, R.U64_MAX)])
    by_term = R.bool_([R.term("all")])
    for q, route in ((everything, WINDOW), (by_term, DRIVER)):
        run(gpu_ctx, [item(main, q, sort, K) for _, _, sort, K in R.sort_cases(main)], route, "sort")


def test_key_layout_pairs(gpu_ctx, main):
    pairs = R.key_pairs(main)
    assert [tb for _, _, tb in pairs][:3] == [64, 65, 146]   # narrow, wide, three words
    for q, route in ((R.bool_([R.term("d30")]), DRIVER), (R.bool_([R.exists("w3")]), WINDOW)):
        items = [item(main, q, R.col_sort(a, o1, (b, o2)), K) for a, b, _ in pairs for o1 in (ASC, DESC)
                 for o2 in (ASC, DESC) for K in (10, 4096)]
        run(gpu_ctx, items, route, "pairs")


def test_small_splits_doc_id_and_column_sorts(gpu_ctx, smalls):
    for q, route in ((R.bool_([R.term("all")]), DRIVER), (R.bool_([R.exists("w3")]), WINDOW)):
        items = [item(sp, q, sort, K) for sp in smalls
                 for sort in (R.SORT_DOC_ASC, R.SORT_DOC_DESC, R.col_sort("w10", ASC), R.col_sort("o10", DESC, ("w64", ASC)))
                 for K in (1, 10, 1000, 4096)]
        run(gpu_ctx, items, route, "small")


def test_paging_through_the_whole_order(gpu_ctx, main):
    """search_after built from the last hit of each page: widths 0, 10, 33, 64, an OPTIONAL column (pages that end on
    a doc without a value: has_v1 = 0), two keys; on k_driver (term-driven) and k_window (range-driven)."""
    for label, q, sort in H.paging_cases(main):
        route = DRIVER if q.children[0].kind == "term" else WINDOW

        def search(sp, q_, sort_, K, sa):
            return run(gpu_ctx, [item(sp, q_, sort_, K, sa)], route, label)[0]
        got = H.page_through(search, main, q, sort, 4096)
        _, want = R.expected(main, q, sort, main.num_docs)
        assert [h[:4] for h in got] == want, label


def test_mixed_batch(gpu_ctx, main, smalls):
    """One call over splits of different widths and cardinalities, per route."""
    for route, mk in ((DRIVER, lambda sp, name, lo, hi: R.bool_([R.term("all"), R.rng(name, lo, hi)])),
                      (WINDOW, lambda sp, name, lo, hi: R.bool_([R.rng(name, lo, hi)]))):
        items = []
        for sp in [main] + smalls + [main]:
            for name in ("w10", "w33", "w64", "o10"):
                c = sp.cols[name]
                lo, hi = (c.min, c.max) if sp.num_docs < 3 else R._wide(sp, name, None)
                items.append(item(sp, mk(sp, name, lo, hi), R.col_sort(name, len(items) % 2), 1000))
        run(gpu_ctx, items, route, "mixed", batch=len(items))


def test_edge_types(gpu_ctx, main):
    """f64 (-inf, -0.0 below 0.0, subnormal, +inf, NaN above +inf), i64, u64 above INT64_MAX, negative datetimes."""
    f = S.f64_to_u64
    fr = [(f(-0.0), f(-0.0)), (f(-0.0), f(0.0)), (f(0.0), f(5e-324)), (f(math.inf), f(math.inf)), (f(math.inf), R.U64_MAX),
          (f(-math.inf), f(-1e-300)), (f(5e-324), f(1.7976931348623157e308)), (f(math.nan), f(math.nan))]
    i = S.i64_to_u64
    ir = [(i(CC.I64_MIN), i(-1)), (i(-1), i(0)), (i(0), i(CC.I64_MAX)), (i(CC.I64_MAX), i(CC.I64_MAX))]
    ur = [((1 << 63), R.U64_MAX), (R.U64_MAX, R.U64_MAX), (0, (1 << 63) - 1)]
    dr = [(0, i(-1)), (i(-1), i(-1)), (i(0), R.U64_MAX)]
    for route, mk in ((DRIVER, lambda r: R.bool_([R.term("d30"), r])), (WINDOW, lambda r: R.bool_([r]))):
        items = []
        for name, rs in (("f64", fr), ("i64", ir), ("u64", ur), ("dt", dr)):
            for k, (lo, hi) in enumerate(rs):
                items.append(item(main, mk(R.rng(name, lo, hi)), R.col_sort(name, k % 2), 1000))
            for o in (ASC, DESC):
                items.append(item(main, mk(R.exists(name)), R.col_sort(name, o, ("i64", 1 - o)), 4096))
        run(gpu_ctx, items, route, "edges")


def test_range_literals_on_the_gpu(gpu_ctx):
    """The QueryAst range literals of the host module, through one GPU leaf request over three splits."""
    docs, parts, imgs = H.literal_splits()
    for im in imgs:
        gpu_ctx.register_split(im)
    try:
        for field, lower, upper in H.LITERAL_RANGES:
            ast = H.range_ast(field, lower, upper)
            out, _ = gpu_root_search(gpu_ctx, imgs, ast, H.LIT_MAPPING, max_hits=len(docs))
            want = H.literal_want(parts, field, lower, upper)
            got = [(int(h["split_id"].rsplit("-", 1)[1]), h["doc_id"]) for h in out["partial_hits"]]
            assert out["num_hits"] == len(want) and got == want, (field, lower, upper)
            cpu = cpu_root_search(imgs, ast, H.LIT_MAPPING, max_hits=len(docs))
            assert out["partial_hits"] == cpu["partial_hits"] and out["num_hits"] == cpu["num_hits"]
    finally:
        for im in imgs:
            gpu_ctx.unregister_split(im.split_id)


def test_device_merge_over_splits_of_different_layouts(gpu_ctx):
    """One qwgpu_leaf_search call over five splits: the same u64 / i64 / f64 fields have a different width, min and gcd
    in each (u: 0..5, >= 2^63, multiples of 1000, absent from one split), and docs miss fields. The merged hits against
    the CPU pipeline and against a brute force over every document, with and without search_after."""
    docs = CC.merge_docs()
    imgs = CC.merge_splits(docs)
    u = [im.columns()[im.column_ord("u")] for im in imgs]
    assert len({(c.bits, c.min_value, c.gcd) for c in u}) == len(imgs)
    for im in imgs:
        gpu_ctx.register_split(im)
    try:
        everything = H.merged_all(docs)
        for sf in H.MERGE_SORTS:
            want = [(s, d) for s, d, _ in H.merge_order(everything, sf[0][0], sf[0][1], sf[1] if len(sf) > 1 else None)]
            for K in (1, 50, len(everything)):
                out, _ = gpu_root_search(gpu_ctx, imgs, {"type": "match_all"}, CC.MERGE_MAPPING, max_hits=K, sort_fields=sf)
                cpu = cpu_root_search(imgs, {"type": "match_all"}, CC.MERGE_MAPPING, max_hits=K, sort_fields=sf)
                assert out["num_hits"] == cpu["num_hits"] == len(everything)
                assert out["partial_hits"] == cpu["partial_hits"], (sf, K)
                assert [(h["split_id"], h["doc_id"]) for h in out["partial_hits"]] == want[:K], (sf, K)
            got, after = [], None
            while True:
                kw = dict(max_hits=97, sort_fields=sf)
                if after is not None:
                    kw["search_after"] = after
                out, _ = gpu_root_search(gpu_ctx, imgs, {"type": "match_all"}, CC.MERGE_MAPPING, **kw)
                cpu = cpu_root_search(imgs, {"type": "match_all"}, CC.MERGE_MAPPING, **kw)
                assert out["partial_hits"] == cpu["partial_hits"], (sf, after)
                page = out["partial_hits"]
                got += [(h["split_id"], h["doc_id"]) for h in page]
                if len(page) < 97:
                    break
                after = dict(page[-1])
            assert got == want, sf
    finally:
        for im in imgs:
            gpu_ctx.unregister_split(im.split_id)
