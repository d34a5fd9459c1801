"""Percentiles aggregations on the GPU (agg_collect_hashed, k_window<COLLECT, true>): the entries of every split equal
percentiles_ref's brute force over the column values exactly (bin, count, min and max of every (node, parent, bin)),
at the top level, under date_histogram and terms > date_histogram, over multi-valued columns, with `missing`, over
negative / zero / positive integers and doubles and at every bit-packed width; a split with more entries than
QWGPU_HASHED_INIT_CELLS goes through the capacity re-run; a batch mixes percentiles plans with dense ones; and
leaf_search over the REST golden's splits returns the golden's values."""
import json

import numpy as np
import pytest

from quickwit_b200 import ffi, plan as P, proto, service, splitgen as S
import percentiles_ref as R
from agg_corpora import Split
from agg_ref import Column, assert_cells, cells
from hashed_ref import assert_entries
from test_oracle_goldens import AGG_MAPPING, AGG_SPLIT1, AGG_SPLIT2

pytestmark = pytest.mark.gpu

HASHED, RETRY, FAST = ffi.KERNEL_HASHED_AGGS, ffi.KERNEL_HASHED_AGGS_RETRY, ffi.KERNEL_FAST_AGGS
HOUR_NS = 3600 * 10**9


def _f64s(xs):
    return np.array([S.f64_to_u64(float(x)) for x in xs], dtype=np.uint64)


def _i64s(xs):
    return np.array([S.i64_to_u64(int(x)) for x in xs], dtype=np.uint64)


def _multi(ctype, values, rng, n, max_per_doc):
    per = rng.integers(0, max_per_doc + 1, size=n)
    start = np.concatenate([[0], np.cumsum(per)]).astype(np.int64)
    return Column(ctype, values(int(start[-1])), start)


def make_split(n, split_id, seed):
    rng = np.random.default_rng(seed)
    ts = np.sort(rng.integers(0, 86_400, n)) * 10**9 + 1_700_000_000 * 10**9
    latf = rng.normal(10, 300, n)
    latf[:6] = [0.0, -0.0, 1e-10, -1e-10, 5e-324, -1e300 / 1e290]
    code = rng.integers(-500, 500, n)
    code[:3] = [0, -1, 1]
    return Split(split_id, n, [
        ("ts", Column(ffi.COL_DATETIME, _i64s(ts))),
        ("svc", Column(ffi.COL_U64, rng.integers(0, 8, n, dtype=np.uint64))),
        ("lat", Column(ffi.COL_U64, np.minimum(rng.lognormal(6, 2, n), 1e7).astype(np.uint64))),
        ("latf", Column(ffi.COL_F64, _f64s(latf))),
        ("code", Column(ffi.COL_I64, _i64s(code))),
        ("latm", _multi(ffi.COL_U64, lambda k: rng.integers(0, 1 << 20, k, dtype=np.uint64), rng, n, 3)),
        ("latmf", _multi(ffi.COL_F64, lambda k: _f64s(rng.normal(0, 1e3, k)), rng, n, 2)),
    ])


def PCT(sp, name, missing=None):
    return P.percentiles(sp.by_name[name], R.num_bins(sp.col(name)), missing)


def T(sp, name, *children):
    return sp.terms(name, children=children)


def DH(sp, *children):
    return sp.hist("ts", float(HOUR_NS), children=children)


def _run(ctx, jobs, docs=None):
    """jobs: [(split, aggs)] in one call; percentiles plans are checked against the brute force, others cell by cell"""
    plans = [P.make_plan(P.bool_([P.match_all()]), 0, aggs=aggs) for _sp, aggs in jobs]
    got = ctx.split_search([sp.img.split_id for sp, _ in jobs], plans)
    for (sp, aggs), plan, r in zip(jobs, plans, got):
        tag = f"{sp.img.split_id} kernel_mask={r.kernel_mask:#x}"
        if service.agg_layout(sp.img, plan)[0]:
            assert r.cells == [] and r.kernel_mask & HASHED, tag
            assert_entries(r.entries, R.entries(plan, sp.cols, docs), tag)
        else:
            assert r.entries == [], tag
            assert_cells(r.cells, cells(aggs, sp.cols), tag)
    return got


@pytest.fixture(scope="module")
def corpora(gpu_ctx):
    c = {"main": make_split(60_001, "pct-main", 1), "small": make_split(1_000, "pct-small", 2)}
    rng = np.random.default_rng(9)
    n = 300_000
    c["retry"] = Split("pct-retry", n, [("svc", Column(ffi.COL_U64, rng.integers(0, 400, n, dtype=np.uint64))),
                                        ("lat", Column(ffi.COL_F64, _f64s(rng.lognormal(0, 4, n) * rng.choice([-1, 1], n))))])
    for sp in c.values():
        gpu_ctx.register_split(sp.img)
    yield c
    for sp in c.values():
        gpu_ctx.unregister_split(sp.img.split_id)


def _trees(sp):
    return {
        "top": [PCT(sp, "lat")],
        "top_signed": [PCT(sp, "latf"), PCT(sp, "code")],
        "under_date_histogram": [DH(sp, PCT(sp, "lat"))],
        "terms_date_histogram": [T(sp, "svc", DH(sp, PCT(sp, "latf"), PCT(sp, "code")))],
        "multi_valued": [PCT(sp, "latm"), T(sp, "svc", PCT(sp, "latmf"))],
        "missing": [PCT(sp, "latm", missing=-3.5), DH(sp, PCT(sp, "latmf", missing=0.0))],
        "siblings": [DH(sp, PCT(sp, "lat"), PCT(sp, "latf")), T(sp, "svc"), PCT(sp, "code")],
    }


@pytest.mark.parametrize("name", ["top", "top_signed", "under_date_histogram", "terms_date_histogram", "multi_valued",
                                  "missing", "siblings"])
def test_entries_equal_brute_force(gpu_ctx, corpora, name):
    for sp in (corpora["main"], corpora["small"]):
        got = _run(gpu_ctx, [(sp, _trees(sp)[name])])
        assert got[0].entries and bool(got[0].kernel_mask & RETRY) == (len(got[0].entries) > ffi.HASHED_INIT_CELLS)


def test_filtered_matches(gpu_ctx, corpora):
    sp = corpora["main"]
    lo, hi = 100, 5000
    plan = P.make_plan(P.bool_([P.range_(sp.img, "lat", lo, hi, occur=ffi.OCCUR_MUST)]), 5, aggs=[DH(sp, PCT(sp, "latf"))])
    r = gpu_ctx.split_search([sp.img.split_id], [plan])[0]
    docs = np.nonzero((sp.col("lat").arr >= lo) & (sp.col("lat").arr <= hi))[0]
    assert_entries(r.entries, R.entries(plan, sp.cols, docs), "filtered")
    assert len(r.hits) == 5


def test_every_bit_packed_width(gpu_ctx):
    rng = np.random.default_rng(21)
    n = 4096
    cols = []
    for b in range(65):
        raw = rng.integers(0, 1 << 64, n, dtype=np.uint64) >> np.uint64(64 - b) if b else np.zeros(n, dtype=np.uint64)
        if b:
            raw[:2] = [0, (1 << b) - 1]
        base = S.i64_to_u64(-(1 << 40)) if b <= 20 else 0  # narrow widths also as i64 values around -2^40
        cols.append((f"w{b}", Column(ffi.COL_I64 if base else ffi.COL_U64, (raw + np.uint64(base)).astype(np.uint64))))
    sp = Split("pct-widths", n, cols)
    assert [sp.img.columns()[sp.by_name[f"w{b}"]].bits for b in range(65)] == list(range(65))
    gpu_ctx.register_split(sp.img)
    try:
        for g in range(0, 65, 8):
            _run(gpu_ctx, [(sp, [PCT(sp, f"w{b}") for b in range(g, min(g + 8, 65))])])
    finally:
        gpu_ctx.unregister_split(sp.img.split_id)


def test_capacity_rerun(gpu_ctx, corpora):
    sp = corpora["retry"]
    got = _run(gpu_ctx, [(sp, [T(sp, "svc", PCT(sp, "lat"))])])
    assert len(got[0].entries) > ffi.HASHED_INIT_CELLS
    assert got[0].kernel_mask & HASHED and got[0].kernel_mask & RETRY, hex(got[0].kernel_mask)


def test_mixed_batch_with_dense_plans(gpu_ctx, corpora):
    """percentiles splits next to dense ones in one call: a fast-path histogram (its raw bounds table shares the staged
    blob with the percentiles tables) and a generic dense tree keep their cells"""
    main, small, other = corpora["main"], corpora["small"], corpora["retry"]
    fast_hist = [main.hist("lat", 5000.0)]
    got = _run(gpu_ctx, [(main, fast_hist), (small, [DH(small, PCT(small, "latf")), PCT(small, "code", missing=1.0)]),
                         (other, [T(other, "svc")])])
    assert got[0].cells and got[2].cells and got[1].entries
    assert got[0].kernel_mask & FAST and got[0].kernel_mask & HASHED, hex(got[0].kernel_mask)
    alone = _run(gpu_ctx, [(main, fast_hist)])
    assert not alone[0].kernel_mask & HASHED and alone[0].cells == got[0].cells


def test_leaf_search_rest_golden(gpu_ctx):
    aggs = {"metrics": {"date_histogram": {"field": "date", "fixed_interval": "30d", "offset": "-4d"},
                        "aggs": {"response": {"percentiles": {"field": "response", "percents": [85], "keyed": False}}}}}
    imgs = [S.build_split(AGG_SPLIT1, AGG_MAPPING, "pct-golden-1"), S.build_split(AGG_SPLIT2, AGG_MAPPING, "pct-golden-2")]
    for img in imgs:
        gpu_ctx.register_split(img)
    try:
        dm = json.dumps(AGG_MAPPING)
        sreq = proto.enc_search_request(json.dumps({"type": "match_all"}), max_hits=0, aggregation_request=json.dumps(aggs))
        lreq = proto.enc_leaf_search_request(sreq, [proto.enc_split_offsets(im.split_id, im.num_docs) for im in imgs], dm)
        resp = proto.dec_leaf_search_response(gpu_ctx.leaf_search(lreq))
        got = json.loads(service.finalize_aggregation(json.dumps(aggs), resp["intermediate_aggregation_result"]))
        b = got["metrics"]["buckets"]
        assert [(x["doc_count"], x["key"]) for x in b] == [(5, 1420070400000.0), (2, 1422662400000.0)]
        assert b[0]["response"] == {"values": [{"key": 85.0, "value": 100.49456770856702}]}
        assert b[1]["response"] == {"values": [{"key": 85.0, "value": 30.26717133872237}]}
    finally:
        for img in imgs:
            gpu_ctx.unregister_split(img.split_id)
