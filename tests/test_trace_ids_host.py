"""find_trace_ids on the host (no GPU): the Python restatement against the reference's own unit vectors, the postcard
bytes, the library's span merge (qwgpu_merge_leaf_responses, finalize) against merge_segment_fruits, request
parsing, and bytes fast fields in the split image."""
import base64
import ctypes
import json
import random

import pytest

from quickwit_b200 import ffi, proto, service, splitgen as S
from pipeline import MATCH_ALL, search_request
import trace_ids_ref as R

MIN = R.I64_MIN


def sid(b: bytes) -> bytes:  # Span::for_test: the bytes, zero padded to 16
    return b + bytes(16 - len(b))


def test_select_trace_ids_reference_vectors():
    sel = R.select_trace_ids
    assert sel([], 0) == [] and sel([], 3) == [] and sel([(0, 0)], 0) == []
    assert sel([(0, 0)], 3) == [(0, 0)]
    assert sel([(0, 1), (0, 0)], 3) == [(0, 1)]
    assert sel([(0, 2), (1, 1), (2, 0)], 3) == [(0, 2), (1, 1), (2, 0)]
    assert sel([(k, 7 - k) for k in range(8)], 3) == [(0, 7), (1, 6), (2, 5)]
    # a boundary tie: the truncation at the 5th span sets the sentinel to 7 and the (2, 7) span is dropped
    assert {o for o, _ in sel([(3, 10), (4, 7), (5, 7), (6, 1), (7, 2), (2, 7)], 2)} == {3, 4}
    # i64::MIN is only kept for the split's first matched doc
    assert sel([(0, MIN), (1, MIN)], 3) == [(0, MIN)]


def test_merge_segment_fruits_reference_vectors():
    m = R.merge_segment_fruits
    foo, bar, qux = sid(b"foo"), sid(b"bar"), sid(b"qux")
    assert m([], 0) == []
    assert m([[(foo, 0), (foo, 1)]], 3) == [(foo, 1)]
    assert m([[(foo, 0), (foo, 1)], [(foo, 1), (foo, 2)]], 3) == [(foo, 2)]
    f3 = [[(foo, 0), (foo, 1), (foo, 2)], [(foo, 2), (bar, 2)], [(foo, 2), (bar, 3)]]
    assert m(f3, 3) == [(bar, 3), (foo, 2)]
    assert m(f3 + [[(qux, 4)]], 3) == [(qux, 4), (bar, 3), (foo, 2)]


def test_postcard_bytes_of_spans():
    assert R.encode_spans([]) == b"\x00"
    assert R.encode_spans([(bytes([255] * 16), MIN)]) == b"\x01" + bytes([255] * 16) + b"\xff" * 9 + b"\x01"
    assert R.encode_spans([(bytes(range(16)), 0), (bytes(16), -1), (bytes(16), 1), (bytes(16), 64)]) == (
        b"\x04" + bytes(range(16)) + b"\x00" + bytes(16) + b"\x01" + bytes(16) + b"\x02" + bytes(16) + b"\x80\x01")
    spans = [(bytes([255] * 16), MIN), (bytes(16), (1 << 63) - 1), (sid(b"x"), 1_700_000_000_123_456_789)]
    assert service.decode_spans(R.encode_spans(spans)) == spans


def _trace_req(n, **kw):
    return search_request(MATCH_ALL, aggs={"num_traces": n, "trace_id_field_name": "trace_id", "span_timestamp_field_name": "ts"}, **kw)


def test_library_merge_and_finalize_agree_with_merge_segment_fruits():
    rng = random.Random(7)
    pool = [bytes(rng.randrange(256) for _ in range(16)) for _ in range(40)]
    for trial in range(60):
        n = rng.choice([0, 1, 2, 5, 20, 100])
        fruits = []
        for _ in range(rng.randint(0, 5)):
            ids = rng.sample(pool, rng.randint(0, 12))
            fruits.append(sorted(((t, rng.choice([MIN, -5, 0, 3, 3, 7, 1 << 40, (1 << 63) - 1])) for t in ids), key=R.span_key))
        # (one response passes through unmerged: the single-response shortcut of collector.rs:922-924)
        want = R.merge_segment_fruits(fruits, n) if len(fruits) > 1 else (fruits[0] if fruits else [])
        req = _trace_req(n)
        resps = [proto.enc_leaf_search_response(num_attempted_splits=1, num_successful_splits=1,
                                                intermediate_aggregation_result=R.encode_spans(f)) for f in fruits]
        if not resps:
            continue
        merged = proto.dec_leaf_search_response(service.merge_leaf_responses(req, resps))
        got = merged["intermediate_aggregation_result"]
        assert got == R.encode_spans(want), trial
        fin = json.loads(service.finalize_aggregation(json.dumps({"num_traces": n, "trace_id_field_name": "trace_id",
                                                                  "span_timestamp_field_name": "ts"}), got))
        assert fin == [{"trace_id": t.hex(), "span_timestamp": ts} for t, ts in want]


DM = {"field_mappings": [{"name": "service", "type": "text", "tokenizer": "raw"},
                         {"name": "trace_id", "type": "bytes", "fast": True, "input_format": "hex"},
                         {"name": "ts", "type": "datetime", "fast": True, "fast_precision": "seconds"},
                         {"name": "dur", "type": "u64", "fast": True}], "timestamp_field": "ts"}


def _img():
    docs = [{"service": "a", "trace_id": bytes([i % 3] * 16).hex(), "ts": 1_700_000_000 + i, "dur": i} for i in range(8)]
    return S.build_split(docs, DM, "trace-host")


def test_trace_request_parsing_and_lowering():
    img = _img()
    dm = json.dumps(DM)
    plan = service.compile_plan(img, _trace_req(7), dm)
    h = ffi.QwPlanHeader.from_buffer_copy(plan)
    assert h.num_aggs == 1 and h.max_hits == 0
    node = ffi.QwAggNode.from_buffer_copy(plan, ctypes.sizeof(ffi.QwPlanHeader) + h.num_nodes * ctypes.sizeof(ffi.QwPlanNode))
    assert node.kind == ffi.AGG_TRACE_IDS and node.num_buckets == 7
    assert node.column == img.column_ord("trace_id") and node.reserved == img.column_ord("ts")
    # an unknown extra key is ignored (serde), a timestamp field absent from the split lowers to ABSENT
    plan = service.compile_plan(img, search_request(MATCH_ALL, aggs={"num_traces": 2, "trace_id_field_name": "trace_id",
                                                                     "span_timestamp_field_name": "nope", "x": 1}), dm)
    node = ffi.QwAggNode.from_buffer_copy(plan, ctypes.sizeof(ffi.QwPlanHeader) + h.num_nodes * ctypes.sizeof(ffi.QwPlanNode))
    assert node.reserved == ffi.ABSENT

    def code(aggs, **kw):
        with pytest.raises(ffi.QwGpuError) as e:
            service.compile_plan(img, search_request(MATCH_ALL, aggs=aggs, **kw), dm)
        return e.value.code

    full = {"num_traces": 3, "trace_id_field_name": "trace_id", "span_timestamp_field_name": "ts"}
    for broken in ({"num_traces": 3}, {**full, "num_traces": "3"}, {**full, "num_traces": -1}, {**full, "num_traces": 2.5},
                   {**full, "trace_id_field_name": 5}, {k: v for k, v in full.items() if k != "span_timestamp_field_name"}):
        assert code(broken) == ffi.EINVALID_AGG, broken
    assert code({**full, "num_traces": 4097}) == ffi.EUNSUPPORTED
    assert code(full, max_hits=10) == ffi.EUNSUPPORTED
    # bytes fields stay out of queries, sorts and tantivy aggregations
    assert code({"t": {"terms": {"field": "trace_id"}}}) == ffi.EUNSUPPORTED
    with pytest.raises(ffi.QwGpuError) as e:
        service.compile_plan(img, search_request({"type": "term", "field": "trace_id", "value": "00"}, max_hits=1), dm)
    assert e.value.code == ffi.EUNSUPPORTED
    with pytest.raises(ffi.QwGpuError) as e:
        service.compile_plan(img, search_request(MATCH_ALL, max_hits=1, sort_fields=[("trace_id", 1)]), dm)
    assert e.value.code == ffi.EUNSUPPORTED


def test_trace_split_order_follows_timestamp_end():
    splits = [proto.enc_split_offsets(f"s{i}", 10, timestamp_start=0, timestamp_end=e) for i, e in enumerate([5, 30, 10])]
    lreq = proto.enc_leaf_search_request(_trace_req(3), splits, json.dumps(DM))
    got = service.optimize_leaf_request(lreq)
    assert [g["split_id"] for g in got] == ["s1", "s2", "s0"] and not any(g["skipped"] for g in got)


@pytest.mark.parametrize("fmt", ["hex", "base64"])
def test_bytes_fast_field_round_trip(fmt):
    rng = random.Random(3)
    vals = [bytes(rng.randrange(256) for _ in range(rng.choice([1, 16, 20]))) for _ in range(30)]
    enc = (lambda b: b.hex()) if fmt == "hex" else (lambda b: base64.b64encode(b).decode())
    docs = [{"b": [enc(v) for v in vals[i:i + (i % 3)]]} for i in range(len(vals))]
    img = S.build_split(docs, {"field_mappings": [{"name": "b", "type": "bytes", "fast": True, "input_format": fmt}]}, "bytes")
    c = img.column_ord("b")
    assert img.columns()[c].type == ffi.COL_BYTES
    assert img.dictionary(c) == sorted({v for i in range(len(vals)) for v in vals[i:i + (i % 3)]})
