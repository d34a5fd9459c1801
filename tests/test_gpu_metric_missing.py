"""`missing` on the stats family on the GPU: every aggregation route against metric_missing_ref's restatement of the
split's result — the dense generic walk (agg_collect_doc) at each of its three levels, with the counters in shared
memory and in global memory, the hashed walk (agg_collect_hashed) with its capacity re-run, and the fast path, which
stays taken for full columns and reports no doc without a value. Counts, min and max are exact, exact sums exact, f64
sums within γ(n-1)·Σ|v| of math.fsum. A 40-split batch mixes plans with and without `missing`, and leaf_search over
JSON requests finalises to the brute force over the documents."""
import json

import numpy as np
import pytest

from quickwit_b200 import ffi, plan as P, proto, service, splitgen as S
import metric_missing_ref as R
from agg_corpora import Split
from agg_ref import Column, assert_cells
from hashed_ref import assert_entries

pytestmark = pytest.mark.gpu

HASHED, RETRY, FAST = ffi.KERNEL_HASHED_AGGS, ffi.KERNEL_HASHED_AGGS_RETRY, ffi.KERNEL_FAST_AGGS
ABSENT = ffi.ABSENT


def _multi(ctype, values, rng, n):
    per = rng.choice([0, 1, 3], size=n, p=[0.3, 0.5, 0.2])
    start = np.concatenate([[0], np.cumsum(per)]).astype(np.int64)
    return Column(ctype, values(int(start[-1])), start)


def _f64s(xs):
    return np.array([S.f64_to_u64(float(x)) for x in xs], dtype=np.uint64)


def make_split(n, split_id, seed, uid=False):
    rng = np.random.default_rng(seed)
    cols = [
        ("svc", Column(ffi.COL_U64, rng.integers(0, 8, n, dtype=np.uint64))),
        ("lvl", _multi(ffi.COL_U64, lambda k: rng.integers(0, 4, k, dtype=np.uint64), rng, n)),
        ("code", Column(ffi.COL_I64, np.array([S.i64_to_u64(int(v)) for v in rng.integers(-20, 20, n)], dtype=np.uint64))),
        ("lat", Column(ffi.COL_U64, rng.integers(0, 5000, n, dtype=np.uint64))),
        ("latf", Column(ffi.COL_F64, _f64s(rng.normal(10, 30, n)))),
        ("vm", _multi(ffi.COL_U64, lambda k: rng.integers(0, 1 << 20, k, dtype=np.uint64), rng, n)),
        ("vmi", _multi(ffi.COL_I64, lambda k: np.array([S.i64_to_u64(int(v)) for v in rng.integers(-10**6, 10**6, k)], dtype=np.uint64), rng, n)),
        ("vmf", _multi(ffi.COL_F64, lambda k: _f64s(rng.normal(0, 1e3, k)), rng, n)),
        ("big", Column(ffi.COL_U64, np.concatenate([[0, 2999], rng.integers(0, 3000, n - 2)]).astype(np.uint64))),
    ]
    if uid:
        cols.append(("uid", Column(ffi.COL_U64, rng.integers(0, 1 << 40, n, dtype=np.uint64))))
    return Split(split_id, n, cols)


def ST(sp, name, missing):
    return P.stats(sp.by_name[name] if name else ABSENT, missing)


def T(sp, name, *children, missing=None):
    return sp.terms(name, children=children, missing=missing)


def H(sp, name, interval, *children):
    return sp.hist(name, interval, children=children)


def _run(ctx, jobs, filt=None):
    """jobs: [(split, aggs)] in one call; each result against the restatement of its layout"""
    plans, docs = [], []
    for sp, aggs in jobs:
        root, d = P.bool_([P.match_all()]), None
        if filt is not None:
            root = P.bool_([P.range_(sp.img, "lat", filt[0], filt[1], occur=ffi.OCCUR_MUST)])
            d = np.nonzero((sp.col("lat").arr >= filt[0]) & (sp.col("lat").arr <= filt[1]))[0]
        plans.append(P.make_plan(root, 0, aggs=aggs))
        docs.append(d)
    got = ctx.split_search([sp.img.split_id for sp, _ in jobs], plans)
    for (sp, aggs), plan, d, r in zip(jobs, plans, docs, got):
        tag = f"{sp.img.split_id} kernel_mask={r.kernel_mask:#x}"
        if service.agg_layout(sp.img, plan)[0]:
            assert r.cells == [] and r.kernel_mask & HASHED, tag
            assert_entries(r.entries, R.device_entries(aggs, sp.cols, d), tag)
        else:
            assert r.entries == [], tag
            assert_cells(r.cells, R.dense_cells(aggs, sp.cols, d), tag)
    return got


@pytest.fixture(scope="module")
def corpora(gpu_ctx):
    rng = np.random.default_rng(17)
    c = {"main": make_split(40_001, "mmg-main", 1), "small": make_split(999, "mmg-small", 2),
         "uid": make_split(70_000, "mmg-uid", 3, uid=True),
         "many": [make_split(int(n), f"mmg-many-{i}", 100 + i) for i, n in enumerate(rng.integers(50, 5000, size=40))]}
    splits = [c["main"], c["small"], c["uid"]] + c["many"]
    for sp in splits:
        gpu_ctx.register_split(sp.img)
    yield c
    for sp in splits:
        gpu_ctx.unregister_split(sp.img.split_id)


def _trees(sp, m=1.0):
    """`m` = None: the same trees without `missing`"""
    mm = (lambda x: None) if m is None else (lambda x: x)
    return {
        "dense_top": [ST(sp, "vm", mm(-1)), ST(sp, "vmf", mm(0.5)), ST(sp, None, mm(3)), ST(sp, "vmi", mm(2.5))],
        "dense_under_bucket": [T(sp, "svc", ST(sp, "vm", mm(0)), ST(sp, None, mm(2))), H(sp, "lat", 700.0, ST(sp, "vmi", mm(-7)))],
        "dense_third_level": [T(sp, "svc", T(sp, "lvl", ST(sp, "vmf", mm(-2.0)), ST(sp, None, mm(1)), missing=9)),
                              H(sp, "code", 5.0, H(sp, "lat", 1000.0, ST(sp, "vm", mm(1e300))))],
        "dense_global_counters": [T(sp, "big", ST(sp, "vm", mm(7)), ST(sp, "vmf", mm(-0.0)))],
        "hashed": [T(sp, "svc", T(sp, "lvl", T(sp, "code", ST(sp, "vm", mm(1)), ST(sp, None, mm(0))), missing=4)),
                   ST(sp, "vmi", mm(-3))],
        "fast_full_columns": [ST(sp, "lat", mm(5)), T(sp, "svc", ST(sp, "latf", mm(-1.5)))],
    }


@pytest.mark.parametrize("name", ["dense_top", "dense_under_bucket", "dense_third_level", "dense_global_counters", "hashed",
                                  "fast_full_columns"])
def test_routes_against_restatement(gpu_ctx, corpora, name):
    for sp in (corpora["main"], corpora["small"]):
        r = _run(gpu_ctx, [(sp, _trees(sp)[name])])[0]
        hashed, fast = bool(r.kernel_mask & HASHED), bool(r.kernel_mask & FAST)
        assert (hashed, fast) == (name == "hashed", name == "fast_full_columns"), hex(r.kernel_mask)


def test_missing_on_a_partial_column_leaves_the_fast_path(gpu_ctx, corpora):
    sp = corpora["main"]
    r = _run(gpu_ctx, [(sp, [ST(sp, "lat", 5), T(sp, "svc", ST(sp, "vm", 1))])])[0]
    assert not r.kernel_mask & FAST and not r.kernel_mask & HASHED, hex(r.kernel_mask)


def test_filtered_matches(gpu_ctx, corpora):
    sp = corpora["main"]
    for name in ("dense_third_level", "hashed"):
        _run(gpu_ctx, [(sp, _trees(sp)[name])], filt=(100, 2500))


def test_hashed_capacity_rerun(gpu_ctx, corpora):
    sp = corpora["uid"]
    got = _run(gpu_ctx, [(sp, [T(sp, "uid", ST(sp, "vm", -1), ST(sp, None, 4))]), (corpora["small"], _trees(corpora["small"])["hashed"])])
    assert len(got[0].entries) > ffi.HASHED_INIT_CELLS
    assert sum(e[3] == ffi.AGG_ENTRY_MISSING for e in got[0].entries) > 70_000
    for r in got:
        assert r.kernel_mask & HASHED and r.kernel_mask & RETRY, hex(r.kernel_mask)


def test_batch_of_40_splits_with_and_without_missing(gpu_ctx, corpora):
    names = ["dense_top", "dense_under_bucket", "dense_third_level", "hashed", "fast_full_columns"]
    jobs = [(sp, _trees(sp, None if i % 3 == 0 else 2.0)[names[i % len(names)]]) for i, sp in enumerate(corpora["many"])]
    got = _run(gpu_ctx, jobs)
    assert all(r.kernel_mask & HASHED for r in got)
    assert sum(bool(r.entries) for r in got) >= 7


# ---- leaf_search from JSON requests ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def json_splits(gpu_ctx):
    rng = np.random.default_rng(23)
    out = []
    for k, n in enumerate((4000, 2500, 1500)):
        absent = k == 2
        docs = R.make_docs(n, rng, absent=absent)
        img = S.build_split(docs, R.mapping(with_absent=not absent), f"mmg-json-{k}")
        gpu_ctx.register_split(img)
        out.append((img, docs))
    yield out
    for img, _docs in out:
        gpu_ctx.unregister_split(img.split_id)


@pytest.mark.parametrize("field,missing", [("u64_optional", 0), ("i64_multi", -3), ("f64_optional", -0.0), ("f64_full", 4.5),
                                           ("datetime_absent", 1_700_000_123 * 10**9), ("bool_multi", 1), ("u64_absent", None)])
def test_leaf_search_json(gpu_ctx, json_splits, field, missing):
    aggs = R.request(field, missing)
    aggs["by_g_avg"] = {"terms": {"field": "g", "order": {"a": "desc"}}, "aggs": {"a": {"avg": {"field": field, "missing": 1e6}}}}
    dm = json.dumps(R.mapping())
    sreq = proto.enc_search_request(json.dumps({"type": "match_all"}), max_hits=0, aggregation_request=json.dumps(aggs))
    lreq = proto.enc_leaf_search_request(sreq, [proto.enc_split_offsets(im.split_id, im.num_docs) for im, _ in json_splits], dm)
    resp = proto.dec_leaf_search_response(gpu_ctx.leaf_search(lreq))
    got = json.loads(service.finalize_aggregation(json.dumps(aggs), resp["intermediate_aggregation_result"]))
    R.check_tree(aggs, got, [d for _im, docs in json_splits for d in docs], ctx=f"{field} missing={missing}")
