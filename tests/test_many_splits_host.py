"""The brute force of test_gpu_many_splits (many_splits_ref.expected) against the CPU pipeline (the oracle per split,
then the product's leaf and root merge) at the same shapes: twins under ids whose lexical, request and registration
orders differ, lists of None values, a single non-empty list, short lists and empty lists, every sort kind. This
validates the reference on machines without a GPU."""
import pytest

from quickwit_b200 import splitgen as S
from quickwit_b200.proto import ASC, DESC
from pipeline import MATCH_ALL, cpu_root_search, term
import many_splits_ref as R

SORTS = [[("_score", DESC)], [("_score", ASC)], [("_doc", ASC)], [("_doc", DESC)], [("c", DESC)], [("c", ASC)],
         [("tenant_id", ASC), ("c", DESC)], [("c", DESC), ("tenant_id", ASC)], [("timestamp", DESC)], [("timestamp", ASC)]]


@pytest.fixture(scope="module")
def bases():
    hand = [R.Base(R.hand_split(n, i, f"hand-{n}", with_c=n != 15_360)) for i, n in enumerate(R.HAND_DOCS)]
    synth = [R.Base(R.synth(i, 1500 + 97 * i)) for i in range(12)]
    return hand, synth, R.Base(R.hand_split(40_000, 12, "hand-solo", solo=True))


def _mixed(bases, n):
    hand, synth, _ = bases
    pool = hand + synth
    return [(sid, pool[i % len(pool)]) for i, sid in R.ids("m", n, 1)]


def _cpu(entries, ast, sort, K, start, **kw):
    imgs = [S.SplitImage(b.img.array, sid) for sid, b in entries]
    return cpu_root_search(imgs, ast, R.MAPPING, max_hits=K - start, start_offset=start, sort_fields=sort, **kw)


def _check(entries, ast, sort, K, start=0, **kw):
    want = _cpu(entries, ast, sort, K, start, **kw)
    nh, got = R.expected(entries, ast, sort, K)
    assert nh == want["num_hits"], (sort, K)
    assert got[start:] == R.hits_of(want), (sort, K, start)


def test_ids_orders_differ():
    pairs = R.ids("m", 33, 1)
    names = [s for _, s in pairs]
    assert sorted(names) != [s for _, s in sorted(pairs)] and names != sorted(names)
    assert dict(R.ids("m", 65, 1))[7] == dict(pairs)[7]


@pytest.mark.parametrize("sort", SORTS, ids=lambda s: "+".join(f"{f}_{'desc' if o else 'asc'}" for f, o in s))
def test_brute_force_matches_cpu_pipeline(bases, sort):
    """Mixed and twin lists at 1 to 65 lists, K on both sides of the list count, with a start offset."""
    hand, synth, _ = bases
    for n in (1, 2, 33, 65):
        mixed = _mixed(bases, n)
        twins = [(sid, hand[-1]) for _, sid in R.ids("w", n, 2)]
        for K, start in ((1, 0), (n, 0), (n + 1, 1), (100, 7), (4097, 0)):
            _check(mixed, term("body", "t1"), sort, K, start)
            if n <= 33:
                _check(twins, term("body", "t0"), sort, K, start)


def test_list_shapes(bases):
    """A single non-empty list, lists shorter than ceil(K / non-empty), every list empty."""
    hand, _, solo = bases
    for n in (33, 65):
        twins = [(sid, hand[-1]) for _, sid in R.ids("w", n, 2)]
        single = list(twins)
        single[n // 2] = ("solo-0", solo)
        for K in (1, 100, 4097):
            _check(single, term("body", "solo"), [("c", DESC)], K)
            _check(twins, term("body", "t2"), [("c", ASC)], K)
            _check(twins, term("body", "t2"), [("_score", DESC)], K)
            _check(_mixed(bases, n), term("body", "absent"), [("c", DESC)], K)


def test_time_range(bases):
    """The request's time range as the brute force restates it: [start_timestamp, end_timestamp)."""
    entries = _mixed(bases, 40)
    tr = (R.T0 + 3 * R.DAY, R.T0 + 8 * R.DAY + 17)
    for sort in ([("timestamp", DESC)], [("c", ASC)]):
        want = _cpu(entries, term("body", "t3"), sort, 300, 0, start_timestamp=tr[0], end_timestamp=tr[1])
        nh, got = R.expected(entries, term("body", "t3"), sort, 300, time_range=tr)
        assert nh == want["num_hits"] > 0 and got == R.hits_of(want)


def test_aggregation_counts(bases):
    entries = _mixed(bases, 40)
    aggs = {"sev": {"terms": {"field": "severity_text"}, "aggs": {"ten": {"terms": {"field": "tenant_id", "size": 200},
                                                                         "aggs": {"d": {"date_histogram": {"field": "timestamp", "fixed_interval": "1d"}}}}}},
            "days": {"date_histogram": {"field": "timestamp", "fixed_interval": "1d"}},
            "ten": {"stats": {"field": "tenant_id"}}}
    a = _cpu(entries, MATCH_ALL, [], 0, 0, aggs=aggs)["aggregations"]
    R.check_aggs(a, [b for _, b in entries])
