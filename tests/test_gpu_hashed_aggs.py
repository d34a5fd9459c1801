"""The hashed aggregation layout on the GPU (agg_collect_hashed in k_window): every case goes through split_search and
is checked against hashed_ref.sparse_cells, the dict brute force computed from the column values — counts, min and
max exact, exact sums exact, f64 sums within γ(n-1)·Σ|v| of math.fsum. Where the dense layout of the same tree is
small enough, the entries are also laid out densely and compared with agg_ref.cells and the CPU oracle. kernel_mask
is asserted on every call: hashed plans take k_window (never k_aggscan), dense plans keep their paths, and corpora
with more distinct cells than QWGPU_HASHED_INIT_CELLS reach the capacity re-run. Finalised JSON through the entries
builder, leaf_search and the root merge equals the JSON of the oracle's dense cells."""
import json

import numpy as np
import pytest

from quickwit_b200 import ffi, plan as P, proto, service, splitgen as S
from oracle import oracle as O
from agg_corpora import Split
from agg_ref import Column, assert_cells, cells
from hashed_ref import assert_entries, entries_to_dense, sparse_cells
import pipeline as PL

pytestmark = pytest.mark.gpu

HASHED, RETRY = ffi.KERNEL_HASHED_AGGS, ffi.KERNEL_HASHED_AGGS_RETRY
WINDOW, AGGSCAN = ffi.KERNEL_WINDOW, ffi.KERNEL_AGGSCAN
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


def _multi(ctype, rng, n, lo, hi, max_per_doc):
    per = rng.integers(0, max_per_doc + 1, size=n)
    start = np.concatenate([[0], np.cumsum(per)]).astype(np.int64)
    return Column(ctype, rng.integers(lo, hi, size=int(start[-1]), dtype=np.uint64), start)


def make_split(n, split_id, seed, uid=False):
    rng = np.random.default_rng(seed)
    wide_vals = np.concatenate([[0, 1 << 63], rng.integers(0, 1 << 63, size=300, dtype=np.uint64)]).astype(np.uint64)
    widei_vals = np.array([S.i64_to_u64(v) for v in [I64_MIN, I64_MAX, -1, 0, 1]] +
                          [S.i64_to_u64(int(v)) for v in rng.integers(I64_MIN, I64_MAX, size=200, dtype=np.int64)], dtype=np.uint64)
    cols = [
        ("svc", Column(ffi.COL_U64, rng.integers(0, 8, size=n, dtype=np.uint64))),
        ("lvl", _multi(ffi.COL_U64, rng, n, 0, 5, 3)),  # 0..3 values per doc: optional and multi-valued
        ("code", Column(ffi.COL_I64, np.array([S.i64_to_u64(int(v)) for v in rng.integers(-50, 50, size=n)], dtype=np.uint64))),
        ("lat", Column(ffi.COL_U64, rng.integers(0, 5000, size=n, dtype=np.uint64))),
        ("latf", Column(ffi.COL_F64, np.array([S.f64_to_u64(float(v)) for v in rng.normal(10, 30, size=n)], dtype=np.uint64))),
        ("latm", _multi(ffi.COL_U64, rng, n, 0, 1 << 20, 2)),
        ("wide", Column(ffi.COL_U64, rng.choice(wide_vals, size=n))),
        ("widei", Column(ffi.COL_I64, rng.choice(widei_vals, size=n))),
    ]
    if uid:
        cols.append(("uid", Column(ffi.COL_U64, rng.integers(0, 1 << 40, size=n, dtype=np.uint64))))
    return Split(split_id, n, cols)


def T(sp, name, *children, missing=None):
    c = sp.col(name)
    nb = ((int(c.arr.max()) - c.min) // c.gcd + 1 if c.num_vals else 0) + (1 if missing is not None else 0)
    return P.Agg(ffi.AGG_TERMS, column=sp.by_name[name], num_buckets=min(nb, 0xFFFFFFFF), children=children, missing=missing)


def H(sp, name, interval, *children, bounds=None):
    return sp.hist(name, interval, bounds=bounds, children=children)


def R(sp, name, ranges, *children):
    return sp.range(name, ranges, children=children)


def ST(sp, name):
    return sp.stats(name)


def _dense_size(aggs):
    from agg_ref import _layout
    return sum(n for *_x, n in _layout(aggs))


def _run(ctx, jobs, max_hits=0, filt=None):
    """jobs: [(split, aggs)] in one call; each result is checked against the brute force of its layout."""
    plans, docs = [], []
    for sp, aggs in jobs:
        if filt is None:
            root, d = P.bool_([P.match_all()]), None
        else:
            lo, hi = filt
            root = P.bool_([P.range_(sp.img, "lat", lo, hi, occur=ffi.OCCUR_MUST)])
            d = np.nonzero((sp.col("lat").arr >= lo) & (sp.col("lat").arr <= hi))[0]
        plans.append(P.make_plan(root, max_hits, aggs=aggs))
        docs.append(d)
    got = ctx.split_search([sp.img.split_id for sp, _ in jobs], plans)
    for (sp, aggs), plan, d, r in zip(jobs, plans, docs, got):
        tag = f"{sp.img.split_id} kernel_mask={r.kernel_mask:#x}"
        hashed, _bound = service.agg_layout(sp.img, plan)
        if hashed:
            assert r.cells == [], tag
            assert_entries(r.entries, sparse_cells(aggs, sp.cols, d), tag)
            if _dense_size(aggs) <= 1 << 20:
                want = cells(aggs, sp.cols, d)
                assert_cells(entries_to_dense(aggs, r.entries), want, f"{tag} laid out densely")
                assert_cells(O.split_search(sp.img, plan).cells, want, f"{tag}: oracle")
        else:
            assert r.entries == [], tag
            assert_cells(r.cells, cells(aggs, sp.cols, d), tag)
        assert r.kernel_mask & WINDOW and not r.kernel_mask & AGGSCAN or not hashed, tag
    return got


@pytest.fixture(scope="module")
def corpora(gpu_ctx):
    rng = np.random.default_rng(3)
    c = {"main": make_split(30_001, "hash-main", 1),
         "many": [make_split(int(n), f"hash-many-{i}", 100 + i) for i, n in enumerate(rng.integers(1, 6000, size=40))],
         "uid": make_split(150_000, "hash-uid", 7, uid=True)}
    c["many"][3] = make_split(31, "hash-many-3", 103)
    splits = [c["main"], c["uid"]] + c["many"]
    for sp in splits:
        gpu_ctx.register_split(sp.img)
    yield c
    for sp in splits:
        gpu_ctx.unregister_split(sp.img.split_id)


def _trees(sp):
    """Depths 3 to 5, every bucket kind at every level, multi-valued / optional columns at inner levels, `missing`."""
    rg = [(0, 100), (100, 100), (50, 4000), (4000, (1 << 64) - 1)]
    return {
        "d3_terms": [T(sp, "svc", T(sp, "lvl", T(sp, "code", ST(sp, "lat")), missing=7))],
        "d3_hist_range": [H(sp, "lat", 700.0, R(sp, "latm", [(0, 1000), (500, 1 << 19), (1 << 19, (1 << 64) - 1)],
                                               H(sp, "code", 10.0, ST(sp, "latf"), ST(sp, "latm"))))],
        "d4_mixed": [R(sp, "lat", rg, T(sp, "lvl", H(sp, "latf", 12.5, T(sp, "svc", ST(sp, "lat")), bounds=(-20.0, 40.0)),
                                       missing=9))],
        "d5": [T(sp, "svc", T(sp, "lvl", R(sp, "code", [(0, S.i64_to_u64(0)), (S.i64_to_u64(-10), (1 << 64) - 1)],
                                          T(sp, "lvl", T(sp, "svc", ST(sp, "latf")), missing=1))))],
        "siblings": [T(sp, "svc", T(sp, "lvl", ST(sp, "lat"), ST(sp, "latf")), H(sp, "lat", 1000.0, T(sp, "code"))),
                     ST(sp, "latm")],
        "wide_u64": [T(sp, "wide", ST(sp, "lat"))],
        "wide_i64": [T(sp, "widei", T(sp, "svc"), ST(sp, "code"))],
    }


@pytest.mark.parametrize("name", ["d3_terms", "d3_hist_range", "d4_mixed", "d5", "siblings", "wide_u64", "wide_i64"])
def test_trees(gpu_ctx, corpora, name):
    sp = corpora["main"]
    got = _run(gpu_ctx, [(sp, _trees(sp)[name])])
    assert got[0].kernel_mask & HASHED and not got[0].kernel_mask & RETRY, hex(got[0].kernel_mask)
    assert got[0].entries


def test_filtered_with_hits(gpu_ctx, corpora):
    sp = corpora["main"]
    got = _run(gpu_ctx, [(sp, _trees(sp)["d4_mixed"])], max_hits=10, filt=(1000, 2500))
    assert got[0].kernel_mask & HASHED and len(got[0].hits) == 10


def test_dense_product_over_2_26(gpu_ctx):
    rng = np.random.default_rng(5)
    n = 20_000
    a = rng.integers(0, 1 << 14, size=n, dtype=np.uint64)
    b = rng.integers(0, 1 << 13, size=n, dtype=np.uint64)
    a[:2], b[:2] = [0, (1 << 14) - 1], [0, (1 << 13) - 1]
    sp = Split("hash-2-26", n, [("a", Column(ffi.COL_U64, a)), ("b", Column(ffi.COL_U64, b)),
                                ("v", Column(ffi.COL_U64, rng.integers(0, 100, size=n, dtype=np.uint64)))])
    gpu_ctx.register_split(sp.img)
    try:
        aggs = [T(sp, "a", T(sp, "b"))]
        assert _dense_size(aggs) > 1 << 26
        got = _run(gpu_ctx, [(sp, aggs)])
        assert got[0].kernel_mask & HASHED
    finally:
        gpu_ctx.unregister_split(sp.img.split_id)


def test_mixed_batch_of_40_splits(gpu_ctx, corpora):
    """40 splits of mixed sizes in one call; every other split takes a hashed tree, the rest a dense one."""
    jobs = []
    for i, sp in enumerate(corpora["many"]):
        t = _trees(sp)
        dense = [T(sp, "svc", T(sp, "lvl", ST(sp, "lat")))]
        jobs.append((sp, t[["d3_terms", "d4_mixed", "d5", "wide_u64"][i % 4]] if i % 2 else dense))
    got = _run(gpu_ctx, jobs)
    assert all(r.kernel_mask & HASHED for r in got)
    assert sum(bool(r.entries) for r in got) >= 19 and sum(bool(r.cells) for r in got) == 20


def test_capacity_rerun(gpu_ctx, corpora):
    sp = corpora["uid"]
    aggs = [T(sp, "uid", T(sp, "svc", ST(sp, "lat")))]
    got = _run(gpu_ctx, [(sp, aggs), (corpora["main"], _trees(corpora["main"])["d3_terms"])])
    assert len(got[0].entries) > ffi.HASHED_INIT_CELLS
    for r in got:
        assert r.kernel_mask & HASHED and r.kernel_mask & RETRY, hex(r.kernel_mask)


def test_capacity_rerun_keeps_fast_histogram(gpu_ctx, corpora):
    """The re-run stages the call's plans again: a dense split whose histogram takes the fast path (a raw-space bounds
    table in the staged blob) must give the same cells in a retried batch as searched alone."""
    uid, main = corpora["uid"], corpora["main"]
    hist = [H(main, "lat", 500.0)]
    both = _run(gpu_ctx, [(uid, [T(uid, "uid", T(uid, "svc", ST(uid, "lat")))]), (main, hist)])
    assert both[1].kernel_mask & RETRY and both[1].kernel_mask & ffi.KERNEL_FAST_AGGS, hex(both[1].kernel_mask)
    alone = _run(gpu_ctx, [(main, hist)])
    assert not alone[0].kernel_mask & RETRY and alone[0].cells
    assert both[1].cells == alone[0].cells


# ---- finalised JSON: entries builder, leaf_search, root merge ---------------------------------------------------------
DM = {"field_mappings": [
    {"name": "svc", "type": "text", "tokenizer": "raw", "fast": True},
    {"name": "lvl", "type": "u64", "fast": True},
    {"name": "code", "type": "i64", "fast": True},
    {"name": "lat", "type": "u64", "fast": True},
    {"name": "latf", "type": "f64", "fast": True},
    {"name": "ts", "type": "datetime", "fast": True, "fast_precision": "seconds"}],
    "timestamp_field": "ts"}


def _docs(n, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        d = {"svc": f"s{int(rng.integers(0, 6))}", "lat": int(rng.integers(0, 5000)), "code": int(rng.integers(-50, 50)),
             "latf": float(rng.normal(10, 3)), "ts": 1_700_000_000 + int(rng.integers(0, 6 * 3600))}
        k = int(rng.integers(0, 4))
        if k:
            d["lvl"] = [int(x) for x in rng.integers(0, 5, size=k)]
        if rng.random() < 0.2:
            del d["svc"]
        out.append(d)
    return out


def _with(agg, **children):
    return {**agg, "aggs": children}


INT_AGGS = {"t": _with({"date_histogram": {"field": "ts", "fixed_interval": "1h"}},
                       s=_with({"terms": {"field": "svc", "size": 3, "missing": "none"}},
                               l=_with({"terms": {"field": "lvl", "size": 2}}, a={"avg": {"field": "lat"}},
                                       c={"stats": {"field": "code"}})))}
F64_AGGS = {"s": _with({"terms": {"field": "svc"}}, l=_with({"terms": {"field": "lvl"}},
                                                          h=_with({"histogram": {"field": "code", "interval": 20}},
                                                                  m={"sum": {"field": "latf"}})))}


@pytest.fixture(scope="module")
def json_splits(gpu_ctx):
    imgs = [S.build_split(_docs(n, 40 + i), DM, split_id=f"hash-json-{i}") for i, n in enumerate((2000, 1, 3500, 777))]
    for img in imgs:
        gpu_ctx.register_split(img)
    yield imgs
    for img in imgs:
        gpu_ctx.unregister_split(img.split_id)


def _close(a, b, path=""):
    if isinstance(a, dict):
        assert a.keys() == b.keys(), path
        for k in a:
            _close(a[k], b[k], f"{path}.{k}")
    elif isinstance(a, list):
        assert len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            _close(x, y, f"{path}[{i}]")
    elif isinstance(a, float) and isinstance(b, float):
        assert abs(a - b) <= 1e-9 * max(1.0, abs(a), abs(b)), f"{path}: {a} vs {b}"
    else:
        assert a == b, f"{path}: {a} vs {b}"


@pytest.mark.parametrize("aggs,exact", [(INT_AGGS, True), (F64_AGGS, False)])
def test_finalised_json(gpu_ctx, json_splits, aggs, exact):
    dm = json.dumps(DM)
    agg_json = json.dumps(aggs)
    req = PL.search_request(PL.MATCH_ALL, max_hits=0, aggs=aggs)
    parts = []
    for img in json_splits:
        plan = service.compile_plan(img, req, dm)
        assert service.agg_layout(img, plan)[0]
        r = gpu_ctx.split_search([img.split_id], [plan])[0]
        assert r.kernel_mask & HASHED
        parts.append(service.build_leaf_response_entries(img, req, dm, r.num_hits, r.hits, r.entries))
    merged = proto.dec_leaf_search_response(service.merge_leaf_responses(req, parts))
    got = json.loads(service.finalize_aggregation(agg_json, merged["intermediate_aggregation_result"]))
    want = PL.cpu_root_search(json_splits, PL.MATCH_ALL, DM, max_hits=0, aggs=aggs)["aggregations"]
    if exact:
        assert got == want
    else:
        _close(got, want)
    # the same request through leaf_search (several splits, one call) and invoke_leaf_search (one response per
    # split: the same intermediate bytes as the entries builder gave above)
    lreq = proto.enc_leaf_search_request(req, [proto.enc_split_offsets(img.split_id, img.num_docs) for img in json_splits], dm)
    leaf = proto.dec_leaf_search_response(gpu_ctx.leaf_search(lreq))
    got2 = json.loads(service.finalize_aggregation(agg_json, leaf["intermediate_aggregation_result"]))
    per = proto.dec_lambda_responses(gpu_ctx.invoke_leaf_search(lreq))
    assert sorted(p["split_id"] for p in per) == sorted(img.split_id for img in json_splits)
    assert all(p["error"] is None for p in per)
    by_id = {p["split_id"]: p["response"] for p in per}
    for img, part in zip(json_splits, parts):
        a = by_id[img.split_id]["intermediate_aggregation_result"]
        b = proto.dec_leaf_search_response(part)["intermediate_aggregation_result"]
        if exact:
            assert a == b  # (f64 sums: atomics add in a different order from call to call)
        else:
            _close(json.loads(service.finalize_aggregation(agg_json, a)), json.loads(service.finalize_aggregation(agg_json, b)))
    if exact:
        assert got2 == want
    else:
        _close(got2, want)


def _multi_split(split_id, seed, docs=100, per_doc=4, num_vals=400):
    """A small split whose multi-valued column gives three nested terms nodes a large bound (num_vals^3 paths)."""
    rng = np.random.default_rng(seed)
    vals = rng.permutation(np.arange(docs * per_doc, dtype=np.uint64) % num_vals)
    start = np.arange(docs + 1, dtype=np.int64) * per_doc
    return Split(split_id, docs, [("m", Column(ffi.COL_U64, vals, start))])


def test_call_budget_refusal(gpu_ctx):
    """The call's hashed tables at their bounds must fit QWGPU_HASHED_MAX_BYTES together: two splits whose tables fit
    one by one but not together are refused with EUNSUPPORTED before any launch; each alone is served."""
    sps = [_multi_split(f"hash-budget-{i}", 60 + i) for i in range(2)]
    for sp in sps:
        gpu_ctx.register_split(sp.img)
    try:
        aggs = {sp.img.split_id: [T(sp, "m", T(sp, "m", T(sp, "m", ST(sp, "m"))))] for sp in sps}
        plans = [P.make_plan(P.bool_([P.match_all()]), 0, aggs=aggs[sp.img.split_id]) for sp in sps]
        for sp, plan in zip(sps, plans):
            hashed, bound = service.agg_layout(sp.img, plan)  # fits alone (no refusal here)
            assert hashed and bound == 400 + 400 ** 2 + 2 * 400 ** 3
        with pytest.raises(ffi.QwGpuError) as e:
            gpu_ctx.split_search([sp.img.split_id for sp in sps], plans)
        assert e.value.code == ffi.EUNSUPPORTED, e.value.msg
        assert "per call" in e.value.msg and str(400 + 400 ** 2 + 2 * 400 ** 3) in e.value.msg
        assert any(sp.img.split_id in e.value.msg for sp in sps)
        for sp in sps:
            got = _run(gpu_ctx, [(sp, aggs[sp.img.split_id])])
            assert got[0].kernel_mask & HASHED and not got[0].kernel_mask & RETRY
    finally:
        for sp in sps:
            gpu_ctx.unregister_split(sp.img.split_id)
