"""Percentiles aggregations on the host (no GPU): the boundary tables against a per-raw-value brute force, the REST
golden and multi-split merges through entries -> leaf response -> leaf merge -> root merge -> finalize, the collapse,
the request's defaults, both `keyed` forms, `missing`, and the refusals."""
import datetime
import json
import math

import numpy as np
import pytest

from quickwit_b200 import ffi, proto, service, splitgen as S
import percentiles_ref as R
import pipeline as PL
from agg_corpora import Split, as_multi
from agg_ref import Column, assert_columns
from test_oracle_goldens import AGG_MAPPING, AGG_SPLIT1, AGG_SPLIT2

GOLDEN_AGGS = {"metrics": {"date_histogram": {"field": "date", "fixed_interval": "30d", "offset": "-4d"},
                           "aggs": {"response": {"percentiles": {"field": "response", "percents": [85], "keyed": False}}}}}


def _mapped(ctype, v):
    if ctype == ffi.COL_DATETIME:
        t = datetime.datetime.fromisoformat(v.replace("Z", "+00:00"))
        return S.i64_to_u64(int(t.timestamp()) * 10**9)
    if ctype == ffi.COL_I64:
        return S.i64_to_u64(int(v))
    if ctype == ffi.COL_F64:
        return S.f64_to_u64(float(v))
    return int(v)


def _doc_columns(img, docs, fields):
    """{column index: Column} of `fields`, built from the documents' values (one or none per doc)"""
    out = {}
    hdr = img.columns()
    for f in fields:
        c = img.column_ord(f)
        if c < 0:
            continue
        vals, start = [], [0]
        for d in docs:
            x = d.get(f)
            for v in (x if isinstance(x, list) else ([] if x is None else [x])):
                vals.append(_mapped(hdr[c].type, v))
            start.append(len(vals))
        out[c] = Column(hdr[c].type, vals, start)
    assert_columns(img, out)
    return out


def _leaf(img, docs, aggs, mapping, fields):
    """the split's leaf response from the brute force's entries"""
    req = PL.search_request(PL.MATCH_ALL, max_hits=0, aggs=aggs)
    dm = json.dumps(mapping)
    plan = service.compile_plan(img, req, dm)
    want = R.entries(plan, _doc_columns(img, docs, fields))
    return req, service.build_leaf_response_entries(img, req, dm, len(docs), [], R.as_entry_list(want))


def _finalize(req, aggs, parts):
    merged = proto.dec_leaf_search_response(service.merge_leaf_responses(req, parts))
    return json.loads(service.finalize_aggregation(json.dumps(aggs), merged["intermediate_aggregation_result"] or b""))


def test_rest_golden_date_histogram_percentiles():
    leaves = []
    for docs, sid in ((AGG_SPLIT1, "agg-1"), (AGG_SPLIT2, "agg-2")):
        img = S.build_split(docs, AGG_MAPPING, sid)
        req, resp = _leaf(img, docs, GOLDEN_AGGS, AGG_MAPPING, ["date", "response"])
        leaves.append(service.merge_leaf_responses(req, [resp]))  # each leaf's merge, then the root's
    got = _finalize(req, GOLDEN_AGGS, leaves)["metrics"]["buckets"]
    assert [(b["doc_count"], b["key"]) for b in got] == [(5, 1420070400000.0), (2, 1422662400000.0)]
    assert got[0]["response"] == {"values": [{"key": 85.0, "value": 100.49456770856702}]}
    assert got[1]["response"] == {"values": [{"key": 85.0, "value": 30.26717133872237}]}


# ---- boundary tables ---------------------------------------------------------------------------------------------
def _f64s(xs):
    return np.array([S.f64_to_u64(float(x)) for x in xs], dtype=np.uint64)


def _i64s(xs):
    return np.array([S.i64_to_u64(int(x)) for x in xs], dtype=np.uint64)


def _neighbours(x, n=3):
    out, lo, hi = [x], x, x
    for _ in range(n):
        lo, hi = math.nextafter(lo, -math.inf), math.nextafter(hi, math.inf)
        out += [lo, hi]
    return out


TINY = [0.0, -0.0, 5e-324, -5e-324, 1e-323, -1e-323, 1.5e-323]
SPECIAL = sorted(set(_neighbours(1e-9) + _neighbours(-1e-9) + TINY + [2.2250738585072014e-308, -2.2250738585072014e-308,
                                                                    1e300, -1e300, 1.0, -1.0, 1e-300, 123.456]))
TABLE_COLUMNS = {
    "u64_small": Column(ffi.COL_U64, np.arange(0, 5000, dtype=np.uint64)),
    "u64_gcd": Column(ffi.COL_U64, np.arange(7, 7 + 13 * 4000, 13, dtype=np.uint64)),
    "i64_cross": Column(ffi.COL_I64, _i64s(range(-3000, 3001))),
    "i64_gcd": Column(ffi.COL_I64, _i64s(range(-9000, 9001, 6))),
    "f64_tiny": Column(ffi.COL_F64, _f64s(TINY)),  # adjacent bit patterns around +-0
    "f64_near_min": Column(ffi.COL_F64, _f64s(_neighbours(1e-9, 40))),
    "f64_near_neg_min": Column(ffi.COL_F64, _f64s(_neighbours(-1e-9, 40))),
    # large raw ranges: every edge and its left neighbour are checked instead
    "u64_wide": Column(ffi.COL_U64, np.array([0, 1, 2, 10**6, 2**40, 2**63, 2**64 - 1], dtype=np.uint64)),
    "i64_wide": Column(ffi.COL_I64, _i64s([-2**63, -10**12, -5, 0, 3, 10**15, 2**63 - 1])),
    "f64_special": Column(ffi.COL_F64, _f64s(SPECIAL)),
    "f64_full": Column(ffi.COL_F64, _f64s([-1.7976931348623157e308, 0.0, 1.7976931348623157e308])),
    "date_ns": Column(ffi.COL_DATETIME, _i64s(np.arange(1_420_070_400, 1_420_070_400 + 86_400 * 30, 3_600) * 10**9)),
    "date_small": Column(ffi.COL_DATETIME, _i64s(range(-1000, 4000, 7))),
}


@pytest.fixture(scope="module")
def table_split():
    n = max(c.num_docs for c in TABLE_COLUMNS.values())
    cols = []
    for name, c in TABLE_COLUMNS.items():
        reps = np.resize(c.arr, n)  # every value at least once
        cols.append((name, Column(c.ctype, reps)))
    return Split("pct-tables", n, cols)


@pytest.mark.parametrize("name", list(TABLE_COLUMNS))
def test_boundary_table_matches_brute_force(table_split, name):
    ci = table_split.by_name[name]
    col = table_split.cols[ci]
    first, edges = service.percentiles_table(table_split.img, ci)
    assert first == R.first_ordinal(col) and len(edges) == R.num_bins(col)
    max_raw = (int(col.arr.max()) - col.min) // col.gcd
    if max_raw <= 200_000:
        assert (first, edges) == R.table_bruteforce(col)
        return
    assert edges[0] == 0
    for i, e in enumerate(edges):
        assert R.ordinal(R.column_f64(col, e)) >= first + i, (i, e)
        if i:
            assert e > 0 and R.ordinal(R.column_f64(col, e - 1)) < first + i, (i, e)
    assert R.ordinal(R.column_f64(col, max_raw)) == first + len(edges) - 1


def test_tables_refuse_nan_and_text():
    sp = Split("pct-nan", 3, [("x", Column(ffi.COL_F64, _f64s([1.0, math.nan, 2.0]))),
                              ("y", Column(ffi.COL_F64, _f64s([1.0, math.inf, 2.0])))])
    for name in ("x", "y"):
        with pytest.raises(ffi.QwGpuError) as e:
            service.percentiles_table(sp.img, sp.by_name[name])
        assert e.value.code == ffi.EUNSUPPORTED


# ---- merges, collapse, request forms -----------------------------------------------------------------------------
MAPPING = {"field_mappings": [{"name": "v", "type": "f64", "fast": True}, {"name": "i", "type": "i64", "fast": True},
                              {"name": "t", "type": "text", "tokenizer": "raw", "fast": True}]}


def _values_split(vals, sid, field="v"):
    docs = [{field: v} if v is not None else {} for v in vals]
    return S.build_split(docs, MAPPING, sid), docs


def _run(splits, aggs, fields=("v", "i")):
    parts = []
    for img, docs in splits:
        req, resp = _leaf(img, docs, aggs, MAPPING, list(fields))
        parts.append(resp)
    return _finalize(req, aggs, parts)


@pytest.mark.parametrize("field", ["v", "i"])
def test_merge_of_three_splits_equals_the_sketch_of_their_union(field):
    rng = np.random.default_rng(11)
    if field == "v":
        chunks = [list(rng.lognormal(3, 2, 400) * rng.choice([-1, 1], 400)) + [0.0, 1e-10, -2e-9],
                  list(rng.uniform(-5, 5, 300)), list(rng.lognormal(8, 1, 200))]
    else:
        chunks = [[int(x) for x in rng.integers(-10**6, 10**6, 400)], [int(x) for x in rng.integers(-50, 50, 300)] + [0, 0],
                  [int(x) for x in rng.integers(0, 10**12, 200)]]
    percents = [0, 0.1, 1, 25, 50, 66.6, 99, 99.9, 100]
    aggs = {"p": {"percentiles": {"field": field, "percents": percents}}}
    got = _run([_values_split(c, f"m{k}", field) for k, c in enumerate(chunks)], aggs)["p"]
    want = R.expected_values(R.sketch_of([float(x) for c in chunks for x in c]), percents)
    assert got == {"values": want}
    assert list(got["values"]) == ["0", "0.1", "1", "25", "50", "66.6", "99", "99.9", "100"]


def test_collapse_of_a_store_spanning_more_than_2048_keys():
    vals = [1e-8, 1e-6, 2.0, 3.0, 1e10, 1e20, 1e30] + [-1e-8, -1e25]
    s = R.sketch_of(vals)
    assert max(s.bins) - min(o for o in s.bins if o > 0) >= 2048
    percents = [1, 10, 20, 30, 40, 50, 60, 70, 80, 90, 99]
    got = _run([_values_split(vals[:4], "c0"), _values_split(vals[4:], "c1")],
               {"p": {"percentiles": {"field": "v", "percents": percents, "keyed": False}}})["p"]
    want = R.expected_values(s, percents, keyed=False)
    assert got == {"values": want}
    # the three smallest positive values share the collapsed floor bin (the largest key - 2047)
    floor = R.value(R.key(1e30) - 2047)
    assert [w["value"] for w in want].count(floor) >= 1 and R.value(R.key(2.0)) not in [w["value"] for w in want]


def test_defaults_keyed_forms_and_missing():
    vals = [3.0, None, 7.5, None, 100.0, 0.25]
    sp = [_values_split(vals, "d0")]
    got = _run(sp, {"p": {"percentiles": {"field": "v"}}})["p"]
    assert got == {"values": R.expected_values(R.sketch_of([3.0, 7.5, 100.0, 0.25]))}
    assert list(got["values"]) == ["1", "5", "25", "50", "75", "95", "99"]
    got = _run(sp, {"p": {"percentiles": {"field": "v", "percents": [50, 99.9], "keyed": False, "missing": -12.5}}})["p"]
    assert got == {"values": R.expected_values(R.sketch_of([3.0, 7.5, 100.0, 0.25, -12.5, -12.5]), [50, 99.9], keyed=False)}
    got = _run(sp, {"p": {"percentiles": {"field": "v", "percents": [0, 100], "missing": 1000}}})["p"]
    assert got == {"values": {"0": 0.25, "100": 1000.0}}
    # a field absent from the split: only `missing`, else an empty sketch (null)
    got = _run(sp, {"p": {"percentiles": {"field": "nope", "percents": [50], "missing": 4}}})["p"]
    assert got == {"values": R.expected_values(R.sketch_of([4.0] * 6), [50])}
    got = _run(sp, {"p": {"percentiles": {"field": "nope", "percents": [50]}}})["p"]
    assert got == {"values": {"50": None}}


def test_empty_histogram_bucket_gives_null():
    docs = [{"v": 1.0, "i": 0}, {"v": 2.0, "i": 100}]
    img = S.build_split(docs, MAPPING, "e0")
    aggs = {"h": {"histogram": {"field": "i", "interval": 50},
                  "aggs": {"p": {"percentiles": {"field": "v", "percents": [50], "keyed": False}}}}}
    got = _run([(img, docs)], aggs)["h"]["buckets"]
    assert [b["p"]["values"][0]["value"] for b in got] == [R.value(R.key(1.0)), None, R.value(R.key(2.0))]


@pytest.mark.parametrize("spec,code", [
    ({"field": "v", "percents": [101]}, ffi.EINVALID_AGG),
    ({"field": "v", "percents": [-0.5]}, ffi.EINVALID_AGG),
    ({"field": "v", "percents": "50"}, ffi.EINVALID_AGG),
    ({"field": "v", "missing": "x"}, ffi.EINVALID_AGG),
    ({"percents": [50]}, ffi.EINVALID_AGG),
    ({"field": "t"}, ffi.EINVALID_AGG),
])
def test_refusals(spec, code):
    img, _docs = _values_split([1.0], "r0")
    img2 = S.build_split([{"v": 1.0, "t": "a"}], MAPPING, "r1")
    req = PL.search_request(PL.MATCH_ALL, max_hits=0, aggs={"p": {"percentiles": spec}})
    with pytest.raises(ffi.QwGpuError) as e:
        service.compile_plan(img2 if spec.get("field") == "t" else img, req, json.dumps(MAPPING))
    assert e.value.code == code


def test_sub_aggregations_and_other_sketches_stay_refused():
    img, _docs = _values_split([1.0], "r2")
    sub = {"p": {"percentiles": {"field": "v"}, "aggs": {"x": {"max": {"field": "v"}}}}}
    with pytest.raises(ffi.QwGpuError) as e:
        service.compile_plan(img, PL.search_request(PL.MATCH_ALL, max_hits=0, aggs=sub), json.dumps(MAPPING))
    assert e.value.code == ffi.EINVALID_AGG
    for t in ("cardinality", "extended_stats", "top_hits"):
        with pytest.raises(ffi.QwGpuError) as e:
            service.compile_plan(img, PL.search_request(PL.MATCH_ALL, max_hits=0, aggs={"x": {t: {"field": "v"}}}), json.dumps(MAPPING))
        assert e.value.code == ffi.EUNSUPPORTED


def test_plan_takes_the_hashed_layout():
    img, _docs = _values_split([1.0, 2.0, 300.0], "h0")
    req = PL.search_request(PL.MATCH_ALL, max_hits=0, aggs={"p": {"percentiles": {"field": "v", "missing": 1}}})
    plan = service.compile_plan(img, req, json.dumps(MAPPING))
    (node,) = R.plan_nodes(plan)
    col = Column(ffi.COL_F64, _f64s([1.0, 2.0, 300.0]))
    assert (node.kind, node.num_buckets, node.has_missing, node.missing_value) == (ffi.AGG_PERCENTILES, R.num_bins(col) + 1, 1, R.f64_bits(1.0))
    assert service.agg_layout(img, plan)[0] is True
