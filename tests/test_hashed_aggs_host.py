"""The hashed aggregation layout on the host (no GPU): which plans take it, the bound on a split's cells and its
refusal, request parsing of deep trees, and the builder from entries — which must give the LeafSearchResponse the
dense builder gives for the same buckets, byte for byte (the oracle's dense cells, turned into entries here)."""
import ctypes as _C
import json

import numpy as np
import pytest

from quickwit_b200 import ffi, plan as P, service, splitgen as S
from oracle import oracle as O
import pipeline as PL
from hashed_ref import dense_to_entries

DM = {"field_mappings": [
    {"name": "svc", "type": "text", "tokenizer": "raw", "fast": True},
    {"name": "lvl", "type": "u64", "fast": True},
    {"name": "code", "type": "i64", "fast": True},
    {"name": "lat", "type": "u64", "fast": True},
    {"name": "latf", "type": "f64", "fast": True},
    {"name": "wide", "type": "u64", "fast": True},
    {"name": "ts", "type": "datetime", "fast": True, "fast_precision": "seconds"}],
    "timestamp_field": "ts"}


def _docs(n, seed):
    rng = np.random.default_rng(seed)
    docs = []
    for i in range(n):
        d = {"svc": f"s{int(rng.integers(0, 6))}", "lat": int(rng.integers(0, 5000)), "latf": float(rng.normal(10, 3)),
             "code": int(rng.integers(-50, 50)), "wide": int(rng.choice([0, 7, 1 << 40, (1 << 63) + 5])),
             "ts": 1_700_000_000 + int(rng.integers(0, 6 * 3600))}
        k = int(rng.integers(0, 4))  # 0..3 values: optional and multi-valued at inner levels
        if k:
            d["lvl"] = [int(x) for x in rng.integers(0, 5, size=k)]
        if rng.random() < 0.2:
            del d["svc"]
        docs.append(d)
    return docs


@pytest.fixture(scope="module")
def split():
    return S.build_split(_docs(3000, 5), DM, split_id="hashed-host")


def _terms(field, size=10, **kw):
    return {"terms": {"field": field, "size": size, **kw}}


def _with(agg, **children):
    out = dict(agg)
    out["aggs"] = children
    return out


CASES = {
    "three_levels": {"t": _with({"date_histogram": {"field": "ts", "fixed_interval": "1h"}},
                                s=_with(_terms("svc", missing="none"), l=_with(_terms("lvl"), a={"avg": {"field": "lat"}})))},
    "inner_cut": {"s": _with(_terms("svc", size=2, segment_size=3),
                             l=_with(_terms("code", size=2, segment_size=4), m={"stats": {"field": "latf"}}))},
    "order_by_metric": {"s": _with(_terms("svc", order={"m.avg": "desc"}),
                                   m={"avg": {"field": "lat"}}, l=_with(_terms("lvl", size=2), x={"max": {"field": "code"}}))},
    "empty_ranges": {"r": _with({"range": {"field": "lat", "ranges": [{"to": 10}, {"from": 10, "to": 10}, {"from": 6000}, {"from": 100}]}},
                                s=_with(_terms("svc"), r2=_with({"range": {"field": "code", "ranges": [{"to": -100}, {"from": 0}]}},
                                                                c={"value_count": {"field": "lat"}})))},
    "hist_bounds": {"h": _with({"histogram": {"field": "lat", "interval": 500, "extended_bounds": {"min": -1000, "max": 9000}}},
                               l=_with({"histogram": {"field": "code", "interval": 10, "min_doc_count": 2}}, s={"sum": {"field": "lat"}}))},
    "five_levels": {"a": _with(_terms("svc", missing="none"), b=_with(_terms("lvl"), c=_with(
        {"histogram": {"field": "code", "interval": 25}}, d=_with(_terms("code", size=3), e={"min": {"field": "latf"}}))))},
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_entries_builder_matches_dense_builder(split, name):
    aggs = CASES[name]
    dm = json.dumps(DM)
    req = PL.search_request(PL.MATCH_ALL, max_hits=0, aggs=aggs)
    plan = service.compile_plan(split, req, dm)
    ref = O.split_search(split, plan)
    dense = service.build_leaf_response(split, req, dm, ref.num_hits, ref.hits, ref.cells)
    tree = _plan_aggs(plan)
    entries = dense_to_entries(tree, ref.cells)
    assert entries, "the case has buckets"
    assert service.build_leaf_response_entries(split, req, dm, ref.num_hits, ref.hits, entries) == dense
    # entry ids carry no order: the same entries with their ids reversed (children before parents)
    n = len(entries)
    rev = [(nd, p if p == ffi.AGG_NO_PARENT else n - 1 - p, k, f, c) for nd, p, k, f, c in reversed(entries)]
    assert service.build_leaf_response_entries(split, req, dm, ref.num_hits, ref.hits, rev) == dense


def _plan_aggs(plan: bytes):
    """P.Agg trees of a compiled plan (dense layout bookkeeping for dense_to_entries)."""
    h = ffi.QwPlanHeader.from_buffer_copy(plan)
    off = C_SIZE_HDR + h.num_nodes * C_SIZE_NODE
    nodes = [ffi.QwAggNode.from_buffer_copy(plan, off + i * C_SIZE_AGG) for i in range(h.num_aggs)]
    objs = [P.Agg(n.kind, column=n.column, num_buckets=n.num_buckets, missing=0 if n.has_missing else None) for n in nodes]
    for i, n in enumerate(nodes):
        objs[i].children = objs[n.first_child:n.first_child + n.num_children]
    return [objs[i] for i, n in enumerate(nodes) if n.parent == 0xFFFFFFFF]


C_SIZE_HDR, C_SIZE_NODE, C_SIZE_AGG = _C.sizeof(ffi.QwPlanHeader), _C.sizeof(ffi.QwPlanNode), _C.sizeof(ffi.QwAggNode)


# ---- selection rule and bound ----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny():
    b = S._Builder(64)
    b.add_column("a", ffi.COL_U64, ffi.CARD_FULL, np.arange(64, dtype=np.uint64) % 8, None)
    b.add_column("m", ffi.COL_U64, ffi.CARD_MULTI, np.arange(100, dtype=np.uint64) % 5,
                 np.minimum(np.arange(65, dtype=np.uint32) * 2, 100).astype(np.uint32))
    return b.finish("hashed-tiny")


def _layout(img, aggs):
    return service.agg_layout(img, P.make_plan(P.bool_([P.match_all()]), 0, aggs=aggs))


def T(nb, *children, col=0, missing=None):
    return P.Agg(ffi.AGG_TERMS, column=col, num_buckets=nb, children=children, missing=missing)


def ST(col=0):
    return P.Agg(ffi.AGG_STATS, column=col)


def test_depth_threshold(tiny):
    assert _layout(tiny, [T(8, T(8, ST()))]) == (False, 0)
    assert _layout(tiny, [T(8, T(8))])[0] is False
    hashed, bound = _layout(tiny, [T(8, T(8, T(8)))])
    assert hashed and bound > 0
    assert _layout(tiny, [T(8, T(8, T(8, ST())))])[0]


def test_dense_cells_threshold(tiny):
    # Σ dense cells 2^26 stays dense, 2^26 + 1 takes the hashed layout
    assert _layout(tiny, [T(1 << 13, T((1 << 13) - 1))])[0] is False
    assert _layout(tiny, [T(1 << 13, T((1 << 13) - 1)), ST()])[0] is True
    assert _layout(tiny, [T(1 << 12, T(1 << 14)), T(1)])[0] is True


def test_terms_space_threshold(tiny):
    assert _layout(tiny, [T(1 << 24)])[0] is False
    assert _layout(tiny, [T((1 << 24) + 1, missing=0)])[0] is False  # the missing slot is not part of the space
    assert _layout(tiny, [T((1 << 24) + 1)])[0] is True
    assert _layout(tiny, [T(0xFFFFFFFF)])[0] is True


def test_bound(tiny):
    # 64 docs, single-valued: min(dense, docs) per node; the multi-valued column (100 values) bounds its chain
    assert _layout(tiny, [T(8, T(8, T(8)))]) == (True, 8 + 64 + 64)
    assert _layout(tiny, [T(8, T(5, T(8, ST()), col=1))]) == (True, 8 + 40 + 100 + 100)
    assert _layout(tiny, [T(0xFFFFFFFF, T(8, ST()))]) == (True, 64 + 64 + 64)


def test_bound_that_does_not_fit_is_refused(tiny):
    deep = [T(0xFFFFFFFF, T(0xFFFFFFFF, T(0xFFFFFFFF, ST(1), col=1), col=1), col=1)]
    # the multi-valued column (100 values) at three levels: at most 100, 100^2, 100^3 paths (and the stats node 100^3)
    assert _layout(tiny, deep) == (True, 100 + 100 ** 2 + 2 * 100 ** 3)
    b = S._Builder(1 << 16)
    b.add_column("m", ffi.COL_U64, ffi.CARD_MULTI, np.arange(1 << 20, dtype=np.uint64),
                 (np.arange((1 << 16) + 1, dtype=np.uint32) * 16).astype(np.uint32))
    big = b.finish("hashed-big")
    with pytest.raises(ffi.QwGpuError) as e:
        _layout(big, [T(0xFFFFFFFF, T(0xFFFFFFFF, T(0xFFFFFFFF, col=0), col=0), col=0)])
    assert e.value.code == ffi.EUNSUPPORTED
    assert "hashed-big" in e.value.msg and str((1 << 20) + (1 << 40) + (1 << 60)) in e.value.msg


def test_wide_terms_lowering_no_longer_refuses(split):
    dm = json.dumps(DM)
    req = PL.search_request(PL.MATCH_ALL, max_hits=0, aggs={"w": _terms("wide")})
    plan = service.compile_plan(split, req, dm)
    (hashed, bound) = service.agg_layout(split, plan)
    assert hashed and bound == split.num_docs
    h = ffi.QwPlanHeader.from_buffer_copy(plan)
    node = ffi.QwAggNode.from_buffer_copy(plan, C_SIZE_HDR + h.num_nodes * C_SIZE_NODE)
    assert node.num_buckets == 0xFFFFFFFF


@pytest.mark.parametrize("depth", range(3, 9))
def test_parse_deep_trees(split, depth):
    agg = {"avg": {"field": "lat"}}
    for i in range(depth - 1):
        agg = _with(_terms("svc" if i % 2 else "lvl"), **{f"n{i}": agg})
    dm = json.dumps(DM)
    plan = service.compile_plan(split, PL.search_request(PL.MATCH_ALL, max_hits=0, aggs={"top": agg}), dm)
    assert ffi.QwPlanHeader.from_buffer_copy(plan).num_aggs == depth
    # terms > terms > avg (3 levels) is the deepest dense tree
    assert service.agg_layout(split, plan)[0] is (depth > 3)


def test_entries_from_the_caller_are_validated(split):
    """qwgpu_build_leaf_response_entries refuses entries outside their node's key space, and repeated buckets."""
    dm = json.dumps(DM)
    for name, node_kind in (("three_levels", ffi.AGG_TERMS), ("empty_ranges", ffi.AGG_RANGE)):
        req = PL.search_request(PL.MATCH_ALL, max_hits=0, aggs=CASES[name])
        plan = service.compile_plan(split, req, dm)
        ref = O.split_search(split, plan)
        tree = _plan_aggs(plan)
        entries = dense_to_entries(tree, ref.cells)
        h = ffi.QwPlanHeader.from_buffer_copy(plan)
        nodes = [ffi.QwAggNode.from_buffer_copy(plan, C_SIZE_HDR + h.num_nodes * C_SIZE_NODE + i * C_SIZE_AGG) for i in range(h.num_aggs)]
        e = next(i for i, x in enumerate(entries) if nodes[x[0]].kind == node_kind and not x[3])
        node, parent, key, flags, cell = entries[e]
        space = nodes[node].num_ranges if node_kind == ffi.AGG_RANGE else nodes[node].num_buckets - nodes[node].has_missing
        bad = [
            entries[:e] + [(node, parent, space + (1 << 20), flags, cell)] + entries[e + 1:],  # beyond the key space
            entries + [entries[e]],                                                          # the same bucket twice
            entries[:e] + [(node, parent, key, 2, cell)] + entries[e + 1:],                  # unknown flag
        ]
        if node_kind == ffi.AGG_RANGE:
            bad.append(entries[:e] + [(node, parent, space, flags, cell)] + entries[e + 1:])
        for b in bad:
            with pytest.raises(ffi.QwGpuError) as err:
                service.build_leaf_response_entries(split, req, dm, ref.num_hits, ref.hits, b)
            assert err.value.code == ffi.EINVALID_ARG, err.value.msg
    # a string column's key beyond its dictionary
    req = PL.search_request(PL.MATCH_ALL, max_hits=0, aggs={"s": _terms("svc")})
    plan = service.compile_plan(split, req, dm)
    ref = O.split_search(split, plan)
    entries = dense_to_entries(_plan_aggs(plan), ref.cells)
    n, p, k, f, c = entries[0]
    with pytest.raises(ffi.QwGpuError) as err:
        service.build_leaf_response_entries(split, req, dm, ref.num_hits, ref.hits, [(n, p, 1000, f, c)])
    assert err.value.code == ffi.EINVALID_ARG
