"""`missing` on avg, sum, min, max, stats and value_count on the host (no GPU): the request's refusals, the compiled
nodes, and leaf build -> merge of three splits -> finalize against metric_missing_ref's brute force over the documents.
The splits' device results are restated from the column values (entries for hashed plans, dense cells with the second
bank otherwise), so these tests exercise the host's fold of count * missing into each metric."""
import json

import numpy as np
import pytest

from quickwit_b200 import ffi, proto, service, splitgen as S
import metric_missing_ref as R
import percentiles_ref as PR
import pipeline as PL
from agg_ref import Column

KINDS = ["stats", "avg", "sum", "min", "max", "value_count"]


def _mapped(field, v):
    t = field.split("_")[0] if "_" in field else {"g": "u64", "ts": "datetime", "h": "i64"}[field]
    if t == "datetime":
        return S.i64_to_u64(int(v) * 10**9)
    if t == "i64":
        return S.i64_to_u64(int(v))
    if t == "f64":
        return S.f64_to_u64(float(v))
    return int(v)


def _columns(img, docs):
    """{column index: Column} of every column of the split, from the documents' values"""
    out = {}
    for f in ["g", "ts", "h"] + R.FIELDS:
        ci = img.column_ord(f)
        if ci < 0:
            continue
        vals, start = [], [0]
        for d in docs:
            x = d.get(f)
            vals += [_mapped(f, v) for v in (x if isinstance(x, list) else ([] if x is None else [x]))]
            start.append(len(vals))
        out[ci] = Column(img.columns()[ci].type, vals, start)
    return out


class Corpus:
    def __init__(self, seed=5, sizes=(180, 150, 120)):
        rng = np.random.default_rng(seed)
        self.splits = []
        for k, n in enumerate(sizes):
            absent = k == len(sizes) - 1
            docs = R.make_docs(n, rng, absent=absent)
            img = S.build_split(docs, R.mapping(with_absent=not absent), f"mm-{seed}-{k}")
            self.splits.append((img, docs, _columns(img, docs)))
        self.docs = [d for _img, docs, _c in self.splits for d in docs]


def leaf(img, docs, cols, aggs, max_hits=0):
    """The split's leaf response from the restated device result of its compiled plan."""
    req = PL.search_request(PL.MATCH_ALL, max_hits=max_hits, aggs=aggs)
    dm = json.dumps(R.mapping())
    plan = service.compile_plan(img, req, dm)
    tops = R.aggs_from_plan(plan)
    if service.agg_layout(img, plan)[0]:
        return req, service.build_leaf_response_entries(img, req, dm, len(docs), [], R.as_entry_list(R.device_entries(tops, cols)))
    dense = service.build_leaf_response(img, req, dm, len(docs), [], [R.cell_tuple(c) for c in R.dense_cells(tops, cols)])
    # the dense cells and the same result as entries build the same response
    assert dense == service.build_leaf_response_entries(img, req, dm, len(docs), [], R.as_entry_list(R.device_entries(tops, cols)))
    return req, dense


def finalize(req, aggs, parts):
    merged = proto.dec_leaf_search_response(service.merge_leaf_responses(req, parts))
    return json.loads(service.finalize_aggregation(json.dumps(aggs), merged["intermediate_aggregation_result"] or b""))


def run(corpus, aggs, splits=None):
    parts, docs = [], []
    for img, ds, cols in (corpus.splits if splits is None else splits):
        req, resp = leaf(img, ds, cols, aggs)
        parts.append(resp)
        docs += ds
    return finalize(req, aggs, parts), docs


@pytest.fixture(scope="module")
def corpus():
    return Corpus()


# ---- the request ------------------------------------------------------------------------------------------------
def _compile(aggs, img=None):
    img = img or S.build_split([{"g": 1, "ts": 1_700_000_000, "h": 0, "f64_full": 1.5}], R.mapping(with_absent=False), "mm-req")
    return service.compile_plan(img, PL.search_request(PL.MATCH_ALL, max_hits=0, aggs=aggs), json.dumps(R.mapping()))


@pytest.mark.parametrize("kind", KINDS + ["count"])
@pytest.mark.parametrize("missing", ["10.0", True, None, {"v": 1}, [1]])
def test_missing_that_is_not_a_number_is_refused(kind, missing):
    with pytest.raises(ffi.QwGpuError) as e:
        _compile({"m": {kind: {"field": "f64_full", "missing": missing}}})
    assert e.value.code == ffi.EINVALID_AGG
    assert f"{kind} `missing` must be a number" in str(e.value)


def test_extended_stats_with_missing_stays_unsupported():
    with pytest.raises(ffi.QwGpuError) as e:
        _compile({"m": {"extended_stats": {"field": "f64_full", "missing": 0}}})
    assert e.value.code == ffi.EUNSUPPORTED


@pytest.mark.parametrize("kind", KINDS + ["count"])
@pytest.mark.parametrize("missing", [0, -0.0, -7, 2.5, 1e300, 9223372036854775807, -9223372036854775808])
def test_compiled_nodes_carry_missing(kind, missing):
    plan = _compile({"m": {kind: {"field": "f64_full", "missing": missing}}, "n": {kind: {"field": "f64_full"}},
                     "t": {"terms": {"field": "g"}, "aggs": {"x": {kind: {"field": "u64_absent", "missing": missing}}}}})
    m, n, t, x = PR.plan_nodes(plan)
    assert (m.kind, m.has_missing, m.missing_value) == (ffi.AGG_STATS, 1, PR.f64_bits(float(missing)))
    assert (n.kind, n.has_missing, n.missing_value) == (ffi.AGG_STATS, 0, 0)
    assert (t.kind, t.has_missing) == (ffi.AGG_TERMS, 0)
    assert (x.kind, x.column, x.has_missing, x.missing_value) == (ffi.AGG_STATS, ffi.ABSENT, 1, PR.f64_bits(float(missing)))


def test_layouts_of_nodes_with_missing():
    """The dense layout gains one cell per parent cell; a deeper tree keeps the hashed layout with one bound entry more
    per parent."""
    img = S.build_split([{"g": g, "ts": 1_700_000_000, "h": 0} for g in range(5)], R.mapping(), "mm-layout")
    dense = _compile({"t": {"terms": {"field": "g"}, "aggs": {"x": {"avg": {"field": "f64_full", "missing": 1}}}}}, img)
    assert service.agg_layout(img, dense)[0] is False
    without = _compile({"t": {"terms": {"field": "g"}, "aggs": {"x": {"avg": {"field": "f64_full"}}}}}, img)
    assert service.agg_layout(img, without)[0] is False
    deep = {"a": {"terms": {"field": "g"}, "aggs": {"b": {"terms": {"field": "h"}, "aggs": {"c": {"terms": {"field": "g"}, "aggs": {
        "x": {"avg": {"field": "f64_full", "missing": 1}}}}}}}}}
    shallow = json.loads(json.dumps(deep))
    del shallow["a"]["aggs"]["b"]["aggs"]["c"]["aggs"]["x"]["avg"]["missing"]
    h1, b1 = service.agg_layout(img, _compile(deep, img))
    h0, b0 = service.agg_layout(img, _compile(shallow, img))
    assert h1 and h0 and b1 == b0 + 5  # one `missing` entry per parent path: the 5 docs reach at most 5


# ---- leaf build -> merge -> finalize --------------------------------------------------------------------------------
@pytest.mark.parametrize("field", R.FIELDS)
def test_every_kind_and_level_against_brute_force(corpus, field):
    t, c = field.split("_")
    missing = {"u64": 0, "i64": -3, "f64": -0.0, "datetime": 1_700_000_123 * 10**9, "bool": 1}[t] if c != "full" else 4.5
    for m in (missing, None):
        aggs = R.request(field, m)
        got, docs = run(corpus, aggs)
        R.check_tree(aggs, got, docs, ctx=f"{field} missing={m}")


@pytest.mark.parametrize("missing", [0, -0.0, -12, 2.5, 1e300, -1e300, 2**62, -(2**63), 2**63])
@pytest.mark.parametrize("field", ["u64_optional", "i64_multi", "f64_optional", "datetime_absent", "bool_multi"])
def test_missing_values(corpus, field, missing):
    aggs = R.request(field, missing, levels=("top", "terms"))
    got, docs = run(corpus, aggs)
    R.check_tree(aggs, got, docs, ctx=f"{field} missing={missing}")


@pytest.mark.parametrize("missing,want_sum", [(-(2**54), 1.0), (-(2**63), None), (-9007199254740992.0, None), (2**63, None)])
def test_integer_missing_joins_the_exact_sum(missing, want_sum):
    """On the exact route an integer `missing` that an i64 holds is added in the 128-bit sum and rounded once: values
    2^53 and 2^53 + 1 and one doc without a value with missing = -2^54 sum to exactly 1 (in f64 after the column's
    sum, 2^54 - 2^54 = 0). 2^63 is past the i64 range: added in f64."""
    docs = [{"g": 0, "ts": 1_700_000_000, "h": 0, "u64_optional": 2**53}, {"g": 0, "ts": 1_700_000_000, "h": 0, "u64_optional": 2**53 + 1},
            {"g": 0, "ts": 1_700_000_000, "h": 0}]
    img = S.build_split(docs, R.mapping(), "mm-exact")
    sp = [(img, docs, _columns(img, docs))]
    aggs = {"s": {"sum": {"field": "u64_optional", "missing": missing}}, "a": {"avg": {"field": "u64_optional", "missing": missing}},
            "t": {"terms": {"field": "g"}, "aggs": {"st": {"stats": {"field": "u64_optional", "missing": missing}}}}}
    got, _docs = run(None, aggs, sp)
    exact = missing != 2**63
    R.check_tree(aggs, got, docs, exact=exact, ctx=f"missing={missing}")
    if want_sum is not None:
        assert got["s"]["value"] == want_sum and got["a"]["value"] == want_sum / 3


def test_absent_column_gives_missing_for_every_doc():
    docs = [{"g": i % 2, "ts": 1_700_000_000 + i, "h": i} for i in range(7)]
    img = S.build_split(docs, R.mapping(with_absent=False), "mm-absent")
    sp = [(img, docs, _columns(img, docs))]
    aggs = {k: {k: {"field": "f64_absent", "missing": -2.5}} for k in KINDS}
    got, _ = run(None, aggs, sp)
    assert got["stats"] == {"avg": -2.5, "count": 7, "max": -2.5, "min": -2.5, "sum": -17.5}
    assert [got[k]["value"] for k in KINDS[1:]] == [-2.5, -17.5, -2.5, -2.5, 7.0]
    got, _ = run(None, {"x": {"avg": {"field": "f64_absent"}}, "c": {"value_count": {"field": "f64_absent"}}}, sp)
    assert got == {"x": {"value": None}, "c": {"value": 0.0}}


@pytest.mark.parametrize("direction", ["desc", "asc"])
def test_terms_ordered_by_avg_with_missing(corpus, direction):
    aggs = {"by_g": {"terms": {"field": "g", "order": {"a": direction}},
                     "aggs": {"a": {"avg": {"field": "f64_optional", "missing": 1e4 if direction == "desc" else -1e4}}}}}
    got, docs = run(corpus, aggs)
    R.check_tree(aggs, got, docs, ctx=direction)
    plain = {"by_g": {"terms": {"field": "g", "order": {"a": direction}}, "aggs": {"a": {"avg": {"field": "f64_optional"}}}}}
    got2, _ = run(corpus, plain)
    R.check_tree(plain, got2, docs, ctx=direction)


def test_requests_without_missing_build_the_same_responses(corpus):
    """A request without `missing` compiles to nodes without it and lays out no second bank: its leaf responses are the
    ones built from agg_ref's cells."""
    from agg_ref import cells
    for img, docs, cols in corpus.splits:
        aggs = R.request("f64_multi", None)
        req = PL.search_request(PL.MATCH_ALL, max_hits=0, aggs=aggs)
        dm = json.dumps(R.mapping())
        plan = service.compile_plan(img, req, dm)
        assert not any(n.has_missing or n.missing_value for n in PR.plan_nodes(plan))
        tops = R.aggs_from_plan(plan)
        old = service.build_leaf_response(img, req, dm, len(docs), [], [R.cell_tuple(c) for c in cells(tops, cols)])
        assert old == leaf(img, docs, cols, aggs)[1]
