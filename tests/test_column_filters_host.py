"""Fast-field range / exists filters and column sort keys on the host: the corpora of column_corpora realise the
column layouts they claim, the oracle agrees with column_ref's brute force on every plan of test_gpu_column_filters,
and QueryAst range literals of every type compile (query_compile.cpp range_query) to the documents a brute force over
the source documents selects."""
import functools
import math

import numpy as np
import pytest

from quickwit_b200 import ffi, splitgen as S
from quickwit_b200.proto import ASC, DESC
from oracle import oracle as O
from pipeline import cpu_root_search
import column_corpora as CC
import column_ref as R


@pytest.fixture(scope="module")
def main():
    return CC.main_split()


@pytest.fixture(scope="module")
def smalls():
    return [CC.small_split(n) for n in CC.SMALL_DOCS]


def _oracle_check(sp, q, sort, K, sa=None, scored=False, aggs=(), ctx=""):
    r = O.split_search(sp.img, R.plan(sp, q, sort, K, sa, aggs))
    R.check(r, sp, q, sort, K, sa, scored, ctx=f"{ctx} {q!r}")
    return r


def test_images_realise_the_column_layouts(main, smalls):
    for sp in [main] + smalls:
        hdr = sp.img.columns()
        for name, c in sp.cols.items():
            h = hdr[sp.ords[name]]
            got = (h.type, h.cardinality, h.num_vals, h.min_value, h.max_value, h.gcd, h.bits)
            want = (c.ctype, c.card, c.num_vals, c.min, c.max, c.gcd, c.bits)
            assert got == want, f"{sp.split_id} {name}: image {got} != {want}"
    for b in range(65):
        assert main.cols[f"w{b}"].bits == b
        assert main.cols[f"w{b}"].gcd == 1 or b == 0
    for b in CC.MC_WIDTHS:
        o, m = main.cols[f"o{b}"], main.cols[f"m{b}"]
        assert (o.card, o.bits, m.card, m.bits) == (ffi.CARD_OPTIONAL, b, ffi.CARD_MULTI, b)
        assert 0 < o.num_vals < CC.N_MAIN and m.start[-1] > CC.N_MAIN and (np.diff(m.start) == 0).any()
        assert not np.all(np.diff(m.start) <= 1)
        # OPTIONAL: both states at the bitmap word edges; MULTI: unsorted values within a doc
        assert {bool(o.has[63]), bool(o.has[64])} == {True, False}
        assert (np.diff(m.vals.astype(object))[np.diff(m.doc_of) == 0] < 0).any() or b == 0
    assert main.cols["g1000"].gcd == 1000 and main.cols["g3"].gcd == 3 and main.cols["g1000"].min == CC.G1000_MIN
    f = set(int(x) for x in main.cols["f64"].vals)
    for v in CC.F64_EDGES:
        assert S.f64_to_u64(v) in f, v
    assert S.f64_to_u64(-0.0) < S.f64_to_u64(0.0) < S.f64_to_u64(5e-324) and S.f64_to_u64(math.inf) < S.f64_to_u64(math.nan)
    assert {S.i64_to_u64(v) for v in CC.I64_EDGES} <= set(int(x) for x in main.cols["i64"].vals)
    assert {CC.U64_MAX, 1 << 63} <= set(int(x) for x in main.cols["u64"].vals)
    assert (main.cols["dt"].vals < np.uint64(1 << 63)).any()
    # the gather's steps: exactly 128 and 129 candidates in one 1024-doc step
    for name, k in (("q128", 128), ("q129", 129)):
        assert np.bincount(main.terms[name] // CC.STEP).max() == k
    assert [(sp.num_docs - 1).bit_length() if sp.num_docs > 1 else 0 for sp in smalls] == [0, 10, 11, 12]


def test_oracle_agrees_with_the_brute_force_on_driver_plans(main):
    for label, q, sort, K in R.driver_cases(main):
        _oracle_check(main, q, sort, K, ctx=label)


def test_oracle_agrees_with_the_brute_force_on_window_plans(main):
    for label, q, sort, K, scored in R.scan_cases(main):
        _oracle_check(main, q, sort, K, scored=scored, ctx=label)
    for label, q, sort, K in R.gather_cases(main):
        _oracle_check(main, q, sort, K, ctx=label)


def test_oracle_agrees_with_the_brute_force_on_sort_keys(main, smalls):
    everything = R.rng("w0", 0, R.U64_MAX)
    for label, name, sort, K in R.sort_cases(main):
        _oracle_check(main, R.bool_([everything]), sort, K, ctx=label)
    for a, b, _ in R.key_pairs(main):
        for o1 in (ASC, DESC):
            for o2 in (ASC, DESC):
                _oracle_check(main, R.bool_([R.term("d30")]), R.col_sort(a, o1, (b, o2)), 1000, ctx=f"pair {a},{b}")
    for sp in smalls:
        for sort in (R.SORT_DOC_ASC, R.SORT_DOC_DESC, R.col_sort("w10", ASC), R.col_sort("o10", DESC, ("w64", ASC))):
            for K in (1, 10, 1000, 4096):
                _oracle_check(sp, R.bool_([R.term("all")]), sort, K, ctx=sp.split_id)


def page_through(search, sp, q, sort, K):
    """Every page of the order, each after the last hit of the page before; returns the concatenated hits."""
    got, sa = [], None
    while True:
        r = search(sp, q, sort, K, sa)
        got += r.hits
        if len(r.hits) < K:
            return got
        sa = R.after(r.hits[-1])


PAGING = [("w0", None), ("w10", None), ("w33", None), ("w64", None), ("o10", None), ("w3", "m9")]


def paging_cases(main):
    for name, second in PAGING:
        for o in (ASC, DESC):
            sort = R.col_sort(name, o, None if second is None else (second, 1 - o))
            for q in (R.bool_([R.term("d30")]), R.bool_([R.rng("w5", 0, R.U64_MAX)])):
                yield f"page {name},{second} {o}", q, sort


def test_oracle_pages_through_the_whole_order(main):
    def search(sp, q, sort, K, sa):
        return _oracle_check(sp, q, sort, K, sa, ctx="page")
    for label, q, sort in paging_cases(main):
        got = page_through(search, main, q, sort, 4096)
        _, want = R.expected(main, q, sort, main.num_docs)
        assert [h[:4] for h in got] == want, label


# ---- range literals, end to end ----------------------------------------------------------------------------------
LIT_MAPPING = {"field_mappings": [{"name": "u", "type": "u64", "fast": True}, {"name": "i", "type": "i64", "fast": True},
                                  {"name": "f", "type": "f64", "fast": True},
                                  {"name": "ts", "type": "datetime", "fast": True, "fast_precision": "seconds"},
                                  {"name": "ms", "type": "datetime", "fast": True, "fast_precision": "milliseconds"},
                                  {"name": "s", "type": "text", "tokenizer": "raw", "fast": True}]}
T0 = 1_700_000_000


def literal_docs():
    rs = np.random.default_rng(41)
    fl = [-math.inf, -1.5, -0.0, 0.0, 1e-300, 2.5, math.inf, -2e10, 7.0]
    words = ["apple", "banana", "cherry", "date", "fig", "grape", "kiwi", "b", "ba", "bananas"]
    pick = lambda xs: xs[int(rs.integers(0, len(xs)))]   # (rs.choice would turn big ints into floats)
    docs = []
    for k in range(500):
        d = {}
        if rs.random() < 0.9:
            d["u"] = pick([0, 1, 5, (1 << 63) - 1, 1 << 63, (1 << 63) + 5, CC.U64_MAX])
        if rs.random() < 0.9:
            d["i"] = pick([CC.I64_MIN, -7, -1, 0, 1, 7, CC.I64_MAX])
        if rs.random() < 0.9:
            d["f"] = pick(fl)
        if rs.random() < 0.9:
            d["ts"] = T0 + int(rs.integers(-3, 4)) + pick([0.0, 0.25, 0.75])   # truncated to the second
        if rs.random() < 0.9:
            d["ms"] = f"2023-11-14T22:13:{20 + int(rs.integers(0, 3)):02d}.{int(rs.integers(0, 1000)):03d}{int(rs.integers(0, 10))}Z"
        if rs.random() < 0.9:
            d["s"] = pick(words)
        docs.append(d)
    return docs


def _stored(field, v):
    """The value of a document as its column holds it (datetime: ns truncated to the field's precision)."""
    if field in ("ts", "ms"):
        prec = 10**9 if field == "ts" else 10**6
        ns = S.parse_datetime_nanos(v)
        return ns - ns % prec
    if field == "f":
        return S.f64_to_u64(v)
    return v


def _bound_value(field, lit):
    if field == "f":
        return S.f64_to_u64(float(lit))
    if field in ("ts", "ms"):
        prec = 10**9 if field == "ts" else 10**6
        ns = S.parse_datetime_nanos(lit)
        return ns - ns % prec
    return lit


LITERAL_RANGES = [
    ("u", {"Included": 1}, {"Excluded": 1 << 63}), ("u", {"Excluded": (1 << 63) - 1}, "Unbounded"),
    ("u", {"Included": 1 << 63}, {"Included": CC.U64_MAX}), ("u", "Unbounded", {"Excluded": 1}),
    ("u", {"Excluded": CC.U64_MAX}, "Unbounded"), ("u", {"Included": str((1 << 63) + 5)}, "Unbounded"),
    ("i", {"Included": -7}, {"Excluded": 0}), ("i", {"Included": CC.I64_MIN}, {"Included": -1}),
    ("i", {"Excluded": -1}, {"Included": CC.I64_MAX}), ("i", "Unbounded", {"Excluded": CC.I64_MIN}),
    ("f", {"Included": "-0.0"}, {"Included": "-0.0"}), ("f", {"Excluded": "-0.0"}, {"Included": 0.0}),
    ("f", {"Included": 0.0}, "Unbounded"), ("f", {"Included": "-inf"}, {"Excluded": "-1.5"}),
    ("f", {"Excluded": 2.5}, {"Included": "inf"}), ("f", "Unbounded", {"Excluded": "-inf"}),
    ("ts", {"Included": "2023-11-14T22:13:19Z"}, {"Excluded": "2023-11-14T22:13:21Z"}),
    ("ts", {"Included": T0 - 1}, {"Included": T0 + 1}), ("ts", {"Excluded": "2023-11-14T22:13:18.5Z"}, "Unbounded"),
    ("ms", {"Included": "2023-11-14T22:13:21.5004Z"}, {"Excluded": "2023-11-14T22:13:22.2Z"}),
    ("ms", "Unbounded", {"Included": "2023-11-14T22:13:20.999999Z"}),
    ("s", {"Included": "b"}, {"Excluded": "cherry"}), ("s", {"Excluded": "banana"}, {"Included": "bananas"}),
    ("s", {"Included": "bb"}, "Unbounded"), ("s", "Unbounded", {"Excluded": "apple"}), ("s", {"Excluded": "kiwi"}, "Unbounded"),
]


def _in_range(field, v, lower, upper):
    x = _stored(field, v)
    for b, is_lo in ((lower, True), (upper, False)):
        if b == "Unbounded":
            continue
        (kind, lit), = b.items()
        y = _bound_value(field, lit)
        if field == "u" and isinstance(y, str):
            y = int(y)
        ok = (x >= y if kind == "Included" else x > y) if is_lo else (x <= y if kind == "Included" else x < y)
        if not ok:
            return False
    return True


def range_ast(field, lower, upper):
    return {"type": "range", "field": field, "lower_bound": lower, "upper_bound": upper}


def literal_splits():
    docs = literal_docs()
    parts = [docs[:200], docs[200:380], docs[380:]]
    return docs, parts, [S.build_split(p, LIT_MAPPING, f"cf-lit-{i}") for i, p in enumerate(parts)]


def literal_want(parts, field, lower, upper):
    """(split index, doc id) of the matches, in the order of a doc-id sort (split id, then doc id, descending)."""
    hits = [(s, d) for s, p in enumerate(parts) for d, doc in enumerate(p) if field in doc and _in_range(field, doc[field], lower, upper)]
    return sorted(hits, reverse=True)


def test_range_literals_end_to_end_against_a_brute_force():
    docs, parts, imgs = literal_splits()
    n_nonempty = 0
    for field, lower, upper in LITERAL_RANGES:
        want = literal_want(parts, field, lower, upper)
        out = cpu_root_search(imgs, range_ast(field, lower, upper), LIT_MAPPING, max_hits=len(docs))
        got = [(int(h["split_id"].rsplit("-", 1)[1]), h["doc_id"]) for h in out["partial_hits"]]
        assert out["num_hits"] == len(want) and got == want, (field, lower, upper, out["num_hits"], len(want))
        n_nonempty += 0 < len(want) < len(docs)
    assert n_nonempty >= len(LITERAL_RANGES) - 6   # (three ranges are empty by construction)


def merge_order(all_docs, field, order, second=None):
    """The leaf merge's order over every document of every split (collector.rs:1120-1153): sort values with None last
    in both directions, then (split id, doc id) in the direction of the first key."""
    def val(d, f):
        if f not in d:
            return None
        return S.f64_to_u64(d[f]) if f == "f" else d[f]

    def cmp_opt(x, y, o):
        if x is None or y is None:
            return (x is not None) - (y is not None)
        return ((x > y) - (x < y)) * (1 if o == DESC else -1)

    def better(a, b):
        c = cmp_opt(val(a[2], field), val(b[2], field), order)
        if c == 0 and second is not None:
            c = cmp_opt(val(a[2], second[0]), val(b[2], second[0]), second[1])
        if c == 0:
            c = ((a[:2] > b[:2]) - (a[:2] < b[:2])) * (1 if order == DESC else -1)
        return c
    return sorted(all_docs, key=functools.cmp_to_key(lambda a, b: -better(a, b)))


MERGE_SORTS = [[("u", DESC)], [("u", ASC)], [("i", ASC), ("u", DESC)], [("f", DESC), ("i", ASC)], [("f", ASC)]]


def merged_all(docs):
    return [(f"cf-merge-{s}", d, doc) for s, part in enumerate(docs) for d, doc in enumerate(part)]


def test_merge_order_against_a_brute_force_over_documents():
    """The CPU leaf / root merge over splits whose fields differ in width, min and gcd, paged with search_after."""
    docs = CC.merge_docs()
    imgs = CC.merge_splits(docs)
    everything = merged_all(docs)
    for sf in MERGE_SORTS:
        want = [(s, d) for s, d, _ in merge_order(everything, sf[0][0], sf[0][1], sf[1] if len(sf) > 1 else None)]
        got, after = [], None
        while True:
            kw = dict(max_hits=97, sort_fields=sf)
            if after is not None:
                kw["search_after"] = after
            out = cpu_root_search(imgs, {"type": "match_all"}, CC.MERGE_MAPPING, **kw)
            assert out["num_hits"] == len(everything)
            page = out["partial_hits"]
            got += [(h["split_id"], h["doc_id"]) for h in page]
            if len(page) < 97:
                break
            after = dict(page[-1])
        assert got == want, sf
