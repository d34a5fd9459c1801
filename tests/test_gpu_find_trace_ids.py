"""find_trace_ids (Jaeger trace search) on the GPU: k_window's collect hook, k_trace_select and k_trace_replay,
through qwgpu_split_search, qwgpu_leaf_search, qwgpu_invoke_leaf_search and the root merge. Every result is compared
bit for bit with the doc-by-doc restatement of SelectTraceIds (tests/trace_ids_ref.py), and with a numpy brute force
(per-trace maximum + lexsort) wherever the N-th and (N+1)-th maxima do not tie."""
import json

import numpy as np
import pytest

from quickwit_b200 import ffi, proto, service, splitgen as S
from pipeline import MATCH_ALL, bool_, search_request, term
import trace_ids_ref as R

pytestmark = pytest.mark.gpu

MIN = R.I64_MIN
DM = {"field_mappings": [{"name": "service", "type": "text", "tokenizer": "raw"},
                         {"name": "trace_id", "type": "bytes", "fast": True},
                         {"name": "ts", "type": "datetime", "fast": True, "fast_precision": "nanoseconds"},
                         {"name": "dur", "type": "u64", "fast": True}], "timestamp_field": "ts"}
SERVICES = [f"svc{i}" for i in range(5)]


class Split:
    """One split built straight from per-doc lists (trace ids, i64 timestamps in ns, service, duration)."""

    def __init__(self, split_id, tids, tss, svc, dur):
        n = len(svc)
        self.tids, self.tss, self.svc, self.dur = tids, tss, svc, dur
        b = S._Builder(n)
        fid = b.add_field("service", 0, ffi.TOK_RAW, None, n)
        svc_arr = np.array(svc)
        for s in sorted(set(svc)):
            b.add_term(fid, s.encode(), np.nonzero(svc_arr == s)[0].astype(np.uint32), None)
        self.dictionary = sorted({t for l in tids for t in l})
        ords = {t: i for i, t in enumerate(self.dictionary)}
        S._column_from_values(b, "trace_id", ffi.COL_BYTES, [[ords[t] for t in l] for l in tids], self.dictionary)
        S._column_from_values(b, "ts", ffi.COL_DATETIME, [[S.i64_to_u64(t) for t in l] for l in tss])
        S._column_from_values(b, "dur", ffi.COL_U64, [[d] for d in dur])
        self.img = b.finish(split_id)
        self.split_id = split_id

    def docs(self, matched):
        """(ordinal, timestamp) of the matched docs in doc order, as the collector reads them."""
        ords = {t: i for i, t in enumerate(self.dictionary)}
        return [(ords[self.tids[d][0]] if self.tids[d] else 0, self.tss[d][0] if self.tss[d] else 0) for d in matched]


def corpus(seed, n_splits, docs_per_split, n_traces, adjacent=True, second_precision=False, multi=False):
    rng = np.random.default_rng(seed)
    pool = [bytes(rng.integers(0, 256, 16, dtype=np.uint8)) for _ in range(n_traces)]
    splits = []
    base = 1_700_000_000 * 10**9
    for s in range(n_splits):
        tids, tss = [], []
        while len(tids) < docs_per_split:
            t = pool[int(rng.zipf(1.3)) % n_traces] if not adjacent else pool[int(rng.integers(0, n_traces))]
            run = int(rng.integers(1, 65)) if adjacent else 1
            start = base + int(rng.integers(0, 3_600 * 10**9))
            for k in range(min(run, docs_per_split - len(tids))):
                ts = start + int(rng.integers(0, 10**9))
                if second_precision:
                    ts -= ts % 10**9
                r = rng.random()
                tids.append([] if r < 0.02 else ([t, pool[int(rng.integers(0, n_traces))]] if multi and r < 0.1 else [t]))
                r = rng.random()
                tss.append([] if r < 0.02 else ([ts, ts - 5] if multi and r < 0.1 else [ts]))
        svc = [SERVICES[min(int(rng.zipf(1.5)) - 1, 4)] for _ in range(docs_per_split)]
        dur = [int(x) for x in rng.integers(0, 1000, docs_per_split)]
        splits.append(Split(f"trace-{seed}-{s}", tids, tss, svc, dur))
    return splits


QUERIES = {
    "match_all": (MATCH_ALL, lambda sp, d: True),
    "term_and_range": (bool_(must=[term("service", "svc0"), {"type": "range", "field": "dur", "lower_bound": {"Included": 100},
                                                                "upper_bound": {"Included": 800}}]),
                       lambda sp, d: sp.svc[d] == "svc0" and 100 <= sp.dur[d] <= 800),
    "must_not": (bool_(must=[MATCH_ALL], must_not=[term("service", "svc1")]), lambda sp, d: sp.svc[d] != "svc1"),
}


def trace_req(ast, n, ts_field="ts"):
    return search_request(ast, aggs={"num_traces": n, "trace_id_field_name": "trace_id", "span_timestamp_field_name": ts_field})


def expected_split(sp, pred, n):
    matched = [d for d in range(len(sp.svc)) if pred(sp, d)]
    return R.split_spans(sp.docs(matched), sp.dictionary, n), matched


def brute_force(sp, matched, n):
    """E: per-trace maximum (i64::MIN only from the first matched doc) + lexsort; None when the boundary ties."""
    docs = sp.docs(matched)
    best = {}
    for i, (o, t) in enumerate(docs):
        if t == MIN and i > 0:
            continue
        best[o] = max(best.get(o, MIN), t)
    if not best:
        return []
    o = np.array(list(best.keys()), dtype=np.int64)
    t = np.array([best[k] for k in best], dtype=np.int64)
    order = np.lexsort((o, -t))
    if len(order) > n > 0 and t[order[n - 1]] == t[order[n]]:
        return None
    return sorted(((sp.dictionary[o[i]], int(t[i])) for i in order[:n]), key=R.span_key)


def u64_to_i64(m):
    v = m ^ (1 << 63)
    return v - (1 << 64) if v >= 1 << 63 else v


def cells_to_spans(sp, cells):
    return sorted(((sp.dictionary[c[1]], u64_to_i64(c[3])) for c in cells if c[0] == 1), key=R.span_key)


def leaf_req(splits, req):
    offsets = [proto.enc_split_offsets(sp.split_id, len(sp.svc)) for sp in splits]
    return proto.enc_leaf_search_request(req, offsets, json.dumps(DM))


def check_corpus(ctx, splits, ns, expect_replay=None):
    for sp in splits:
        ctx.register_split(sp.img)
    replays = 0
    dm = json.dumps(DM)
    for qname, (ast, pred) in QUERIES.items():
        for n in ns:
            req = trace_req(ast, n)
            want = []
            for sp in splits:
                exp, matched = expected_split(sp, pred, n)
                want.append(exp)
                plan = service.compile_plan(sp.img, req, dm)
                got = ctx.split_search([sp.split_id], [plan])[0]
                assert got.kernel_mask & ffi.KERNEL_TRACE_SELECT and got.kernel_mask & ffi.KERNEL_WINDOW
                replays += bool(got.kernel_mask & ffi.KERNEL_TRACE_REPLAY)
                assert cells_to_spans(sp, got.cells) == exp, (qname, n, sp.split_id)
                e = brute_force(sp, matched, n)
                if e is not None:
                    assert exp == e, (qname, n, sp.split_id)
            merged = R.merge_segment_fruits(want, n)
            # seam A: every split in one call, leaf merge on the host
            leaf = ctx.leaf_search(leaf_req(splits, req))
            dec = proto.dec_leaf_search_response(leaf)
            assert dec["num_successful_splits"] == len(splits) and not dec.get("failed_splits")
            assert dec["intermediate_aggregation_result"] == R.encode_spans(merged), (qname, n)
            # seam B: one result per split
            per = proto.dec_lambda_responses(ctx.invoke_leaf_search(leaf_req(splits, req)))
            by_id = {p["split_id"]: p["response"]["intermediate_aggregation_result"] for p in per}
            for sp, w in zip(splits, want):
                assert by_id[sp.split_id] == R.encode_spans(w)
            # root merge of two leaves
            if len(splits) > 1:
                h = len(splits) // 2
                parts = [ctx.leaf_search(leaf_req(splits[:h], req)), ctx.leaf_search(leaf_req(splits[h:], req))]
                root = proto.dec_leaf_search_response(service.merge_leaf_responses(req, parts))
                assert root["intermediate_aggregation_result"] == R.encode_spans(merged), (qname, n)
                fin = json.loads(service.finalize_aggregation(json.dumps({"num_traces": n, "trace_id_field_name": "trace_id",
                                                                          "span_timestamp_field_name": "ts"}),
                                                              root["intermediate_aggregation_result"]))
                assert fin == [{"trace_id": t.hex(), "span_timestamp": ts} for t, ts in merged]
    if expect_replay is not None:
        assert (replays > 0) == expect_replay, replays


def test_adjacent_traces_across_splits(gpu_ctx):
    check_corpus(gpu_ctx, corpus(1, 3, 30_000, 3_000), [0, 1, 20, 1000, 4096])


def test_interleaved_multivalued_with_missing_values(gpu_ctx):
    check_corpus(gpu_ctx, corpus(2, 2, 20_000, 1_500, adjacent=False, multi=True), [1, 20, 1000])


def test_more_traces_than_4096(gpu_ctx):
    check_corpus(gpu_ctx, corpus(3, 1, 60_000, 12_000, adjacent=False), [1000, 4096])


def test_second_precision_ties_take_the_replay(gpu_ctx):
    check_corpus(gpu_ctx, corpus(4, 2, 30_000, 4_000, adjacent=False, second_precision=True), [1, 20, 1000], expect_replay=True)


def _one_split(ctx, split_id, rows):
    ids = [bytes([k]) * 16 for k in range(256)]
    sp = Split(split_id, [[ids[o]] for o, _ in rows], [[t] for _, t in rows], ["svc0"] * len(rows), [0] * len(rows))
    ctx.register_split(sp.img)
    return sp, ids


def test_boundary_tie_vector_returns_the_reference_traces(gpu_ctx):
    sp, ids = _one_split(gpu_ctx, "trace-tie-vector", [(3, 10), (4, 7), (5, 7), (6, 1), (7, 2), (2, 7)])
    got = gpu_ctx.split_search([sp.split_id], [service.compile_plan(sp.img, trace_req(MATCH_ALL, 2), json.dumps(DM))])[0]
    assert got.kernel_mask & ffi.KERNEL_TRACE_REPLAY
    assert {t for t, _ in cells_to_spans(sp, got.cells)} == {ids[3], ids[4]}


def test_i64_min_only_for_the_first_matched_doc(gpu_ctx):
    sp, ids = _one_split(gpu_ctx, "trace-min-vector", [(0, MIN), (1, MIN)])
    got = gpu_ctx.split_search([sp.split_id], [service.compile_plan(sp.img, trace_req(MATCH_ALL, 3), json.dumps(DM))])[0]
    assert cells_to_spans(sp, got.cells) == [(ids[0], MIN)]


def test_absent_timestamp_column_reads_zero_and_missing_trace_column_fails_the_split(gpu_ctx):
    sp, ids = _one_split(gpu_ctx, "trace-no-ts", [(1, 5), (2, 9), (1, 3)])
    req = trace_req(MATCH_ALL, 5, ts_field="other_ts")
    got = gpu_ctx.split_search([sp.split_id], [service.compile_plan(sp.img, req, json.dumps(DM))])[0]
    assert cells_to_spans(sp, got.cells) == [(ids[1], 0), (ids[2], 0)]
    bad = search_request(MATCH_ALL, aggs={"num_traces": 5, "trace_id_field_name": "nope", "span_timestamp_field_name": "ts"})
    dec = proto.dec_leaf_search_response(gpu_ctx.leaf_search(leaf_req([sp], bad)))
    assert dec["failed_splits"] and dec["num_successful_splits"] == 0
