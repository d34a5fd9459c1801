"""The partial-result cache key on the host (CacheKey::from_split_meta_and_request and HalfOpenRange,
quickwit-search/src/leaf_cache.rs:98-185), through `qwgpu_leaf_cache_keys`.

The reference's own cases (`test_leaf_search_cache_no_timestamp`, `test_leaf_search_cache_timestamp`,
leaf_cache.rs:251-440) are restated as key equalities: a `get` that hits after a `put` is the same key, a `get` that
misses is another key. What a hit returns, the LRU and the counters need a device: tests/test_gpu_leaf_cache.py.

HalfOpenRange is reached here through the two ranges it is built from on the wire: the request's
[start_timestamp, end_timestamp) and the split's [timestamp_start, timestamp_end]. Neither has an excluded start, so
the rule "an excluded start of i64::MAX is empty" is not reachable from a request."""
import json

from quickwit_b200 import proto, service

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
DM = json.dumps({"field_mappings": [{"name": "body", "type": "text"},
                                    {"name": "timestamp", "type": "datetime", "fast": True}],
                 "timestamp_field": "timestamp"})
Q_TEST = json.dumps({"type": "term", "field": "body", "value": "test"})
Q_TEST2 = json.dumps({"type": "term", "field": "body", "value": "test2"})
MATCH_ALL = json.dumps({"type": "match_all"})


def split(split_id, ts_start=None, ts_end=None, num_docs=0):
    return proto.enc_split_offsets(split_id, num_docs, timestamp_start=ts_start, timestamp_end=ts_end)


def keys(query, splits, doc_mapper=DM, **kw):
    """{split_id: row} of qwgpu_leaf_cache_keys for one LeafSearchRequest."""
    sreq = proto.enc_search_request(query, index_id_patterns=("test-idx",), **kw)
    rows = service.leaf_cache_keys(proto.enc_leaf_search_request(sreq, splits, doc_mapper))
    return {r["split_id"]: r for r in rows}


def key(query, one_split, **kw):
    (row,) = keys(query, [one_split], **kw).values()
    assert row["looked_up"]
    return row["key"]


def test_no_timestamp():
    """test_leaf_search_cache_no_timestamp: a put of (split_1, query_1) is found by the same pair only."""
    s1, s2 = split("split_1"), split("split_2")
    k11 = key(Q_TEST, s1, max_hits=10)
    assert key(Q_TEST, s1, max_hits=10) == k11
    assert key(Q_TEST, s2, max_hits=10) != k11      # another split
    assert key(Q_TEST2, s1, max_hits=10) != k11     # another query
    assert keys(Q_TEST, [s1], max_hits=10)["split_1"]["range"] == [I64_MIN, None]


def test_timestamp():
    """test_leaf_search_cache_timestamp: windows that cover the split key alike, windows that cut it do not."""
    s1 = split("split_1", 100, 199)
    s2 = split("split_2", 150, 249)
    s3 = split("split_3", 150, 249)
    q1 = dict(start_timestamp=100, end_timestamp=250, max_hits=10)
    q1bis = dict(start_timestamp=150, end_timestamp=300, max_hits=10)
    q2 = dict(max_hits=10)
    q2bis = dict(start_timestamp=50, end_timestamp=200, max_hits=10)
    # split_1: 1 and 1bis cover different parts of it
    assert key(Q_TEST, s1, **q1) != key(Q_TEST, s1, **q1bis)
    # split_2: 1 and 1bis both cover all of it
    assert key(Q_TEST, s2, **q1) == key(Q_TEST, s2, **q1bis)
    # split_1: 2 and 2bis both cover all of it
    assert key(Q_TEST2, s1, **q2) == key(Q_TEST2, s1, **q2bis)
    # split_2: 2 covers all of it, 2bis only a part
    assert key(Q_TEST2, s2, **q2) != key(Q_TEST2, s2, **q2bis)
    # split_3: a put of the bounded request is not found by the unbounded one, and is found by itself
    assert key(Q_TEST2, s3, **q2bis) != key(Q_TEST2, s3, **q2)
    assert key(Q_TEST2, s3, **q2bis) == key(Q_TEST2, s3, **q2bis)
    # the merged ranges themselves
    assert keys(Q_TEST, [s1], **q1)["split_1"]["range"] == [100, 200]
    assert keys(Q_TEST, [s1], **q1bis)["split_1"]["range"] == [150, 200]
    assert keys(Q_TEST, [s2], **q1)["split_2"]["range"] == [150, 250]
    assert keys(Q_TEST, [s2], **q2bis)["split_2"]["range"] == [150, 200]


def test_changed_max_hits_misses():
    s1 = split("split_1", 100, 199)
    assert key(Q_TEST, s1, max_hits=10) != key(Q_TEST, s1, max_hits=11)
    assert key(Q_TEST, s1, max_hits=10) != key(Q_TEST, s1, max_hits=10, start_offset=1)
    assert key(Q_TEST, s1, max_hits=10) != key(Q_TEST, s1, max_hits=10, sort_fields=[("timestamp", proto.DESC)])


def test_count_hits_does_not_matter():
    """At the scale of one split every hit is counted: CountAll and Underestimate key alike."""
    s1 = split("split_1", 100, 199)
    for kw in (dict(max_hits=10), dict(max_hits=10, start_timestamp=120, end_timestamp=150)):
        assert key(Q_TEST, s1, count_hits=0, **kw) == key(Q_TEST, s1, count_hits=1, **kw)
    aggs = json.dumps({"n": {"value_count": {"field": "timestamp"}}})
    assert key(Q_TEST, s1, aggregation_request=aggs, count_hits=0) == key(Q_TEST, s1, aggregation_request=aggs, count_hits=1)


def test_doc_mapper_is_part_of_the_key():
    s1 = split("split_1", 100, 199)
    other = json.dumps({**json.loads(DM), "field_mappings": json.loads(DM)["field_mappings"] + [{"name": "x", "type": "u64", "fast": True}]})
    assert key(Q_TEST, s1, max_hits=10) != key(Q_TEST, s1, doc_mapper=other, max_hits=10)


def test_key_is_taken_after_the_split_rewrite():
    """A match-all request sorted by split id keeps hits on the splits it needs only. The others are demoted to
    count-only requests, and a count-only match-all without time range or aggregation is answered from the split's
    metadata: it is never looked up. Under CountHits::Underestimate a split with nothing left to compute is skipped."""
    splits = [split(f"s{i}", 0, 99, num_docs=100) for i in range(3)]
    rows = keys(MATCH_ALL, splits, max_hits=10)
    # s2 sorts first (split ids descending) and keeps its hits; s1 and s0 are demoted
    assert {k: r["looked_up"] for k, r in rows.items()} == {"s2": True, "s1": False, "s0": False}
    assert rows["s2"]["key"] == keys(MATCH_ALL, [splits[2]], max_hits=10)["s2"]["key"]
    # with a time range nothing is demoted, and every split is looked up with the request as sent
    rows = keys(MATCH_ALL, splits, max_hits=10, start_timestamp=0)
    assert [r["looked_up"] for r in rows.values()] == [True] * 3
    assert len({r["key"] for r in rows.values()}) == 3
    rows = keys(MATCH_ALL, splits, max_hits=0)
    assert [r["looked_up"] for r in rows.values()] == [False] * 3
    rows = keys(Q_TEST, splits, max_hits=0, count_hits=1)
    assert [r["looked_up"] for r in rows.values()] == [False] * 3


def test_half_open_range_edges():
    # an included split end of i64::MAX is unbounded
    assert keys(Q_TEST, [split("a", 5, I64_MAX)], max_hits=1)["a"]["range"] == [5, None]
    assert keys(Q_TEST, [split("a", I64_MIN, I64_MAX)], max_hits=1)["a"]["range"] == [I64_MIN, None]
    assert keys(Q_TEST, [split("a", I64_MAX, I64_MAX)], max_hits=1)["a"]["range"] == [I64_MAX, None]
    assert keys(Q_TEST, [split("a", I64_MIN, I64_MIN)], max_hits=1)["a"]["range"] == [I64_MIN, I64_MIN + 1]
    assert keys(Q_TEST, [split("a", I64_MAX - 1, I64_MAX - 1)], max_hits=1)["a"]["range"] == [I64_MAX - 1, I64_MAX]
    # request ranges at the limits
    assert keys(Q_TEST, [split("a")], max_hits=1, start_timestamp=I64_MAX)["a"]["range"] == [I64_MAX, None]
    assert keys(Q_TEST, [split("a")], max_hits=1, start_timestamp=I64_MIN)["a"]["range"] == [I64_MIN, None]
    assert keys(Q_TEST, [split("a")], max_hits=1, end_timestamp=I64_MAX)["a"]["range"] == [I64_MIN, I64_MAX]
    assert keys(Q_TEST, [split("a", 0, I64_MAX)], max_hits=1, start_timestamp=I64_MAX, end_timestamp=I64_MAX)["a"]["range"] == [0, 0]
    # every empty range is 0..0, so all empty windows key alike
    empties = [dict(end_timestamp=I64_MIN), dict(start_timestamp=I64_MAX, end_timestamp=I64_MAX),
               dict(start_timestamp=500, end_timestamp=400), dict(start_timestamp=7, end_timestamp=7)]
    for kw in empties:
        assert keys(Q_TEST, [split("a")], max_hits=1, **kw)["a"]["range"] == [0, 0], kw
    assert len({key(Q_TEST, split("a"), max_hits=1, **kw) for kw in empties}) == 1
    # a window that misses the split is empty as well, and keys like the empty window
    s = split("a", 100, 199)
    assert keys(Q_TEST, [s], max_hits=1, start_timestamp=200, end_timestamp=300)["a"]["range"] == [0, 0]
    assert key(Q_TEST, s, max_hits=1, start_timestamp=200, end_timestamp=300) == key(Q_TEST, s, max_hits=1, end_timestamp=50)
    # an end of 100 excludes the split's first second; 101 keeps it
    assert keys(Q_TEST, [s], max_hits=1, end_timestamp=100)["a"]["range"] == [0, 0]
    assert keys(Q_TEST, [s], max_hits=1, end_timestamp=101)["a"]["range"] == [100, 101]
