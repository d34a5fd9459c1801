"""`ip` fields on the host: the address parser against Rust's `IpAddr::from_str` vectors, the reference's golden
documents through the CPU oracle, range edge cases, field shapes, every refusal, and terms aggregations keyed by
address (leaf intermediates, the merge over splits whose dictionaries differ, finalisation) against the brute force
in ip_ref.py. CPU only; test_gpu_ip_fields.py runs the same requests on the device."""
import ipaddress
import json
import random

import pytest

from quickwit_b200 import ffi, proto, service, splitgen as S
from quickwit_b200.proto import ASC, DESC
from pipeline import MATCH_ALL, bool_, cpu_root_search, cpu_split_response, full_text, search_request, term
import ip_ref as R

# ---- the golden documents: quickwit-search/src/tests.rs:1451-1628 -------------------------------------------------
GOLDEN_DOCS = [{"log": "User not found", "host": "192.168.0.1"}, {"log": "Request failed", "host": "10.10.12.123"},
               {"log": "Request successful", "host": "10.10.11.125"}, {"log": "Auth service error", "host": "2001:db8::1:0:0:1"},
               {"log": "Settings saved", "host": "::afff:4567:890a"}, {"log": "Request failed", "host": "10.10.12.123"}]
GOLDEN_INDEXED = {"field_mappings": [{"name": "log", "type": "text"}, {"name": "host", "type": "ip"}],
                  "default_search_fields": ["log"]}
GOLDEN_FAST = {"field_mappings": [{"name": "log", "type": "text"}, {"name": "host", "type": "ip", "fast": True}],
               "default_search_fields": ["log"]}


def rng_q(field, lo=None, hi=None, lo_incl=True, hi_incl=True):
    b = lambda v, inc: "Unbounded" if v is None else {("Included" if inc else "Excluded"): v}
    return {"type": "range", "field": field, "lower_bound": b(lo, lo_incl), "upper_bound": b(hi, hi_incl)}


def exists_q(field):
    return {"type": "field_presence", "field": field}


def term_set_q(field, values):
    return {"type": "term_set", "terms_per_field": {field: list(values)}}


def doc_ids(res):
    return sorted(h["doc_id"] for h in res["partial_hits"])


def run(imgs, ast, dm, **kw):
    kw.setdefault("max_hits", 1000)
    return cpu_root_search(imgs if isinstance(imgs, list) else [imgs], ast, dm, **kw)


def error_code(imgs, ast, dm, **kw):
    with pytest.raises(ffi.QwGpuError) as e:
        run(imgs, ast, dm, **kw)
    return e.value.code, e.value.msg


# ---- the address parser ------------------------------------------------------------------------------------------
ACCEPTED = [("192.168.0.1", "::ffff:192.168.0.1"), ("2001:db8::1:0:0:1", "2001:db8::1:0:0:1"),
            ("::afff:4567:890a", "::afff:4567:890a"), ("127.0.0.1", "::ffff:127.0.0.1"),
            ("2001:db8:85a3::8a2e:370:7334", "2001:db8:85a3::8a2e:370:7334"), ("::", "::"),
            ("ffff:ffff:ffff:ffff:ffff:ffff:ffff:ffff", "ffff:ffff:ffff:ffff:ffff:ffff:ffff:ffff"),
            ("2001:0db8:0000:0000:0000:0000:0000:0001", "2001:db8::1"), ("2001:DB8::1", "2001:db8::1"),
            ("::1.2.3.4", "::102:304"), ("1:2:3:4:5:6:1.2.3.4", "1:2:3:4:5:6:102:304"), ("1::", "1::"),
            ("1:2:3:4:5:6:7::", "1:2:3:4:5:6:7:0"), ("0.0.0.0", "::ffff:0.0.0.0")]
REJECTED = ["01.2.3.4", "256.0.0.1", "1.2.3", "fe80::1%eth0", "[::1]", "::1:2:3:4:5:6:7:8", "1.2.3.4 ", " 1.2.3.4",
            "1.2.3.4:80", "1.2.3.4.5", "", ":::", "1:::2", "::1::", "12345::", "1:2:3:4:5:6:7:8:9", "1.2.3.4::",
            "1:2:3:4:5:6:7:1.2.3.4", "::ffff:01.2.3.4", "g::1"]


@pytest.mark.parametrize("text,canonical", ACCEPTED)
def test_parser_accepts(text, canonical):
    assert S.parse_ip(text) == R.v6(canonical).packed


def test_full_form_equals_compressed_form():
    assert S.parse_ip("2001:0db8:0000:0000:0000:ff00:0042:8329") == S.parse_ip("2001:db8::ff00:42:8329")


@pytest.mark.parametrize("text", REJECTED)
def test_parser_rejects(text):
    with pytest.raises(ValueError):
        S.parse_ip(text)


def test_rendering_matches_brute_force():
    rnd = random.Random(7)
    samples = [t for t, _ in ACCEPTED] + ["::1", "1::1", "1:0:0:1:0:0:0:1", "0:0:1:0:0:1:0:0", "1:0:1:0:1:0:1:0"]
    for _ in range(2000):
        groups = [rnd.choice([0, 0, 0, 1, 0xffff, rnd.randrange(1 << 16)]) for _ in range(8)]
        samples.append(":".join(format(g, "x") for g in groups))
    for t in samples:
        assert S.format_ip(S.parse_ip(t)) == R.render(R.v6(t)), t


# ---- goldens -----------------------------------------------------------------------------------------------------
def test_golden_indexed_term():
    img = S.build_split(GOLDEN_DOCS, GOLDEN_INDEXED, "golden")
    assert img.columns() == [] and img.field_names() == ["log", "host"]
    assert run(img, MATCH_ALL, GOLDEN_INDEXED, max_hits=10)["num_hits"] == 6
    for mode in ("bool", "phrase_fallback_to_intersection"):
        res = run(img, full_text("host", "10.10.11.125", mode=mode), GOLDEN_INDEXED, max_hits=10)
        assert res["num_hits"] == 1 and doc_ids(res) == [2]
    assert doc_ids(run(img, term("host", "10.10.12.123"), GOLDEN_INDEXED)) == [1, 5]
    assert doc_ids(run(img, term("host", "::ffff:10.10.12.123"), GOLDEN_INDEXED)) == [1, 5]


def test_golden_fast_range():
    img = S.build_split(GOLDEN_DOCS, GOLDEN_FAST, "golden")
    res = run(img, rng_q("host", "10.0.0.0", "10.255.255.255"), GOLDEN_FAST, max_hits=10)
    assert res["num_hits"] == 3 and doc_ids(res) == [1, 2, 5]
    assert doc_ids(run(img, full_text("host", "10.10.11.125"), GOLDEN_FAST)) == [2]


# ---- a random corpus ---------------------------------------------------------------------------------------------
def addresses(n, seed):
    """n distinct addresses: IPv4 (mapped), pure IPv6, and the edges of the IPv4-mapped block"""
    rnd = random.Random(seed)
    out = {"::", "::fffe:ffff:ffff", "::1:0:0:0", "ffff:ffff:ffff:ffff:ffff:ffff:ffff:ffff", "0.0.0.0", "255.255.255.255"}
    while len(out) < n:
        if rnd.random() < 0.6:
            out.add(".".join(str(rnd.randrange(256)) for _ in range(4)))
        else:
            out.add(R.render(ipaddress.IPv6Address(rnd.getrandbits(128) >> rnd.choice([0, 64, 96]))))
    return sorted(out)


def corpus(num_docs, seed, pool, multi=True, p_missing=0.1):
    rnd = random.Random(seed)
    docs = []
    for d in range(num_docs):
        doc = {"log": rnd.choice(["alpha beta", "beta gamma", "gamma", "alpha"]), "ts": 1_700_000_000 + rnd.randrange(86_400),
               "status": rnd.randrange(5)}
        r = rnd.random()
        if r >= p_missing:
            k = rnd.choice([1, 1, 1, 2, 3]) if multi else 1
            vs = [rnd.choice(pool) for _ in range(k)]
            doc["client_ip"] = vs[0] if k == 1 else vs
        docs.append(doc)
    return docs


def mapping(indexed=True, fast=True):
    return {"field_mappings": [{"name": "log", "type": "text", "record": "freq", "fieldnorms": True},
                               {"name": "client_ip", "type": "ip", "indexed": indexed, "fast": fast},
                               {"name": "ts", "type": "datetime", "fast": True, "fast_precision": "seconds"},
                               {"name": "status", "type": "u64", "fast": True}],
            "timestamp_field": "ts"}


POOL = addresses(40, 1)
DOCS = corpus(600, 2, POOL)
DM = mapping()


@pytest.fixture(scope="module")
def img():
    return S.build_split(DOCS, DM, "ip-main")


def test_image_layout(img):
    c = img.columns()[img.column_ord("client_ip")]
    assert c.type == ffi.COL_IP and c.cardinality == ffi.CARD_MULTI
    present = sorted({a for doc in DOCS for a in R.values(doc, "client_ip")})
    assert img.dictionary(img.column_ord("client_ip")) == [a.packed for a in present]
    f = img.fields()[img.field_names().index("client_ip")]
    assert f.tokenizer == ffi.TOK_IP and f.flags == 0 and f.num_terms == len(present)


def test_bad_value_fails_the_build():
    with pytest.raises(ValueError):
        S.build_split([{"client_ip": "10.0.0.1"}, {"client_ip": "10.0.0.256"}], DM, "bad")
    with pytest.raises(ValueError):
        S.build_split([{"client_ip": ["10.0.0.1", "host.example"]}], mapping(indexed=True, fast=False), "bad")


def test_dynamic_mode_never_infers_ip():
    img = S.build_split([{"x": "10.0.0.1"}], {"mode": "dynamic"}, "dyn")
    assert img.columns()[img.column_ord("x")].type == ffi.COL_STR


RANGES = [("10.0.0.0", "10.255.255.255", True, True), (None, None, True, True), ("::", None, True, True),
          ("0.0.0.0", "255.255.255.255", True, True), ("0.0.0.0", "255.255.255.255", False, False),
          (None, "::ffff:0.0.0.0", True, False), ("::1:0:0:0", None, False, True), ("8000::", None, True, True),
          ("ffff:ffff:ffff:ffff:ffff:ffff:ffff:ffff", None, False, True), (None, "::", True, False),
          ("::ffff:7f00:1", "127.0.0.1", True, True), ("200.0.0.0", "100.0.0.0", True, True)]


def _ranges_with_dictionary_bounds():
    """bounds on, between, below and above the dictionary's entries, included and excluded"""
    ps = sorted(R.v6(a) for a in POOL)
    out = list(RANGES)
    for i in (0, 5, len(ps) // 2, len(ps) - 1):
        a = ps[i]
        out.append((str(a), str(a), True, True))
        out.append((str(a), str(a), False, True))
        out.append((str(a), None, False, True))
        out.append((None, str(a), True, False))
        if i + 1 < len(ps):
            mid = ipaddress.IPv6Address((int(a) + int(ps[i + 1])) // 2)
            out.append((str(mid), str(ps[-1]), True, True))
            out.append((None, str(mid), True, True))
    return out


@pytest.mark.parametrize("lo,hi,lo_incl,hi_incl", _ranges_with_dictionary_bounds())
def test_range_against_brute_force(img, lo, hi, lo_incl, hi_incl):
    got = doc_ids(run(img, rng_q("client_ip", lo, hi, lo_incl, hi_incl), DM))
    assert got == R.range_docs(DOCS, "client_ip", lo, hi, lo_incl, hi_incl)


def test_ipv4_range_leaves_pure_ipv6_out(img):
    got = doc_ids(run(img, rng_q("client_ip", "0.0.0.0", "255.255.255.255"), DM))
    assert all(any(a.ipv4_mapped is not None for a in R.values(DOCS[d], "client_ip")) for d in got)
    assert any(all(a.ipv4_mapped is None for a in R.values(doc, "client_ip")) and R.values(doc, "client_ip") for doc in DOCS)


@pytest.mark.parametrize("shape", ["fast+indexed", "fast-only", "indexed-only"])
def test_terms_and_sets_every_shape(shape):
    dm = mapping(indexed=shape != "fast-only", fast=shape != "indexed-only")
    img = S.build_split(DOCS, dm, "shape")
    probes = POOL[:6] + ["10.1.2.3", "::ffff:" + POOL[0] if "." in POOL[0] else "1::2"]
    for a in probes:
        assert doc_ids(run(img, term("client_ip", a), dm)) == R.term_docs(DOCS, "client_ip", a), a
        assert doc_ids(run(img, full_text("client_ip", a), dm)) == R.term_docs(DOCS, "client_ip", a), a
    want = sorted(set(R.term_docs(DOCS, "client_ip", POOL[1])) | set(R.term_docs(DOCS, "client_ip", POOL[7])))
    assert doc_ids(run(img, term_set_q("client_ip", [POOL[1], POOL[7], "1.1.1.1"]), dm)) == want
    # beside a BM25 clause, sorted by doc id (the ip clause is never scored)
    q = bool_(must=[full_text("log", "alpha")], filter=[term("client_ip", POOL[3])])
    want = [d for d in R.term_docs(DOCS, "client_ip", POOL[3]) if "alpha" in DOCS[d]["log"].split()]
    assert doc_ids(run(img, q, dm)) == want
    if shape != "indexed-only":
        assert doc_ids(run(img, exists_q("client_ip"), dm)) == R.exists_docs(DOCS, "client_ip")
        assert doc_ids(run(img, rng_q("client_ip", POOL[2], POOL[20]), dm)) == R.range_docs(DOCS, "client_ip", POOL[2], POOL[20])
    else:
        code, msg = error_code(img, rng_q("client_ip", POOL[2], POOL[20]), dm)
        assert code == ffi.EINVALID_QUERY and "only supported for fast fields" in msg


def test_field_absent_from_split():
    docs = [{"log": "alpha", "status": 1}, {"log": "beta", "status": 2}]
    for indexed, fast in ((True, True), (False, True), (True, False)):
        dm = mapping(indexed=indexed, fast=fast)
        img = S.build_split(docs, dm, "absent")
        assert run(img, term("client_ip", "10.0.0.1"), dm)["num_hits"] == 0
        if fast:
            assert run(img, rng_q("client_ip", "10.0.0.0", None), dm)["num_hits"] == 0
        assert run(img, exists_q("client_ip"), dm)["num_hits"] == 0
        assert error_code(img, term("client_ip", "10.0.0"), dm)[0] == ffi.EINVALID_QUERY


# ---- refusals ----------------------------------------------------------------------------------------------------
def test_refusals(img):
    E = ffi
    assert error_code(img, term("client_ip", "not-an-ip"), DM)[0] == E.EINVALID_QUERY
    assert error_code(img, full_text("client_ip", "10.0.0.1 10.0.0.2"), DM)[0] == E.EINVALID_QUERY
    assert error_code(img, rng_q("client_ip", "10.0.0", None), DM)[0] == E.EINVALID_QUERY
    assert error_code(img, {"type": "wildcard", "field": "client_ip", "value": "10.*"}, DM)[0] == E.EINVALID_QUERY
    assert error_code(img, {"type": "regex", "field": "client_ip", "regex": "10.*"}, DM)[0] == E.EINVALID_QUERY
    assert error_code(img, {"type": "phrase_prefix", "field": "client_ip", "phrase": "10.0"}, DM)[0] == E.EINVALID_QUERY
    # scored: refused under _score ranking, served in a filter or under any other sort
    scored = [("_score", DESC)]
    for q in (term("client_ip", POOL[0]), term_set_q("client_ip", POOL[:2]), bool_(should=[full_text("log", "alpha"), term("client_ip", POOL[0])])):
        assert error_code(img, q, DM, sort_fields=scored)[0] == E.EUNSUPPORTED
    q = bool_(must=[full_text("log", "alpha")], filter=[term("client_ip", POOL[0])])
    assert run(img, q, DM, sort_fields=scored)["num_hits"] == len([d for d in R.term_docs(DOCS, "client_ip", POOL[0]) if "alpha" in DOCS[d]["log"].split()])
    assert run(img, rng_q("client_ip", "10.0.0.0", None), DM, sort_fields=scored)["num_hits"] == len(R.range_docs(DOCS, "client_ip", "10.0.0.0", None))
    code, msg = error_code(img, MATCH_ALL, DM, sort_fields=[("client_ip", ASC)])
    assert code == E.EINVALID_ARG and msg == "Unsupported sort field type `IpAddr`."
    for agg in ({"histogram": {"field": "client_ip", "interval": 10}}, {"range": {"field": "client_ip", "ranges": [{"to": 5}]}},
                {"stats": {"field": "client_ip"}}, {"avg": {"field": "client_ip"}}, {"percentiles": {"field": "client_ip"}},
                {"composite": {"sources": [{"ip": {"terms": {"field": "client_ip"}}}]}}):
        assert error_code(img, MATCH_ALL, DM, max_hits=0, aggs={"a": agg})[0] == E.EUNSUPPORTED, agg
    for missing in ("nope", 5, "10.0.0"):
        assert error_code(img, MATCH_ALL, DM, max_hits=0, aggs={"a": {"terms": {"field": "client_ip", "missing": missing}}})[0] == E.EINVALID_AGG


# ---- terms aggregations ------------------------------------------------------------------------------------------
def split_set(n_splits, seed):
    """splits whose dictionaries differ: each draws from its own slice of a shared pool"""
    pool = addresses(60, seed)
    rnd = random.Random(seed)
    out = []
    for i in range(n_splits):
        lo = rnd.randrange(0, 30)
        docs = corpus(rnd.randrange(50, 300), seed * 100 + i, pool[lo:lo + 25])
        out.append((docs, S.build_split(docs, DM, f"ip-{seed}-{i:03d}")))
    return out


AGG_SPECS = [({}, "_count", True), ({"order": {"_key": "asc"}}, "_key", False), ({"order": {"_key": "desc"}}, "_key", True),
             ({"order": {"_count": "asc"}}, "_count", False), ({"size": 3}, "_count", True), ({"size": 100}, "_count", True),
             ({"missing": "10.0.0.1"}, "_count", True), ({"missing": "::1", "order": {"_key": "asc"}}, "_key", False),
             ({"min_doc_count": 5}, "_count", True)]


def terms_request(extra):
    return {"ips": {"terms": {"field": "client_ip", "split_size": 1000, **extra}}}


@pytest.mark.parametrize("extra,order,desc", AGG_SPECS)
@pytest.mark.parametrize("n_splits", [1, 5])
def test_terms_against_brute_force(extra, order, desc, n_splits):
    splits = split_set(n_splits, 3 + n_splits)
    q = rng_q("status", 1, 3)
    res = run([img for _, img in splits], q, DM, max_hits=0, aggs=terms_request(extra))
    matched = [(docs, [d for d in range(len(docs)) if 1 <= docs[d]["status"] <= 3]) for docs, _ in splits]
    counts = R.terms_counts(matched, "client_ip", extra.get("missing"))
    want = R.terms_result(counts, extra.get("size", 10), order, desc, extra.get("min_doc_count", 1))
    assert res["aggregations"]["ips"] == want


def test_leaf_intermediate_merge_order_is_free():
    """per-split leaf intermediates merged in any order and grouping finalise to the same result"""
    splits = split_set(6, 11)
    req = search_request(MATCH_ALL, max_hits=0, aggs=terms_request({"size": 50}))
    parts = [cpu_split_response(img, req, DM) for _, img in splits]
    agg = json.dumps(terms_request({"size": 50}))

    def fin(merged):
        return json.loads(service.finalize_aggregation(agg, proto.dec_leaf_search_response(merged)["intermediate_aggregation_result"]))
    a = fin(service.merge_leaf_responses(req, parts))
    b = fin(service.merge_leaf_responses(req, [service.merge_leaf_responses(req, parts[3:]), service.merge_leaf_responses(req, parts[:3][::-1])]))
    assert a == b
    counts = R.terms_counts([(docs, range(len(docs))) for docs, _ in splits], "client_ip")
    assert a["ips"] == R.terms_result(counts, 50)


def test_terms_nested_under_date_histogram():
    splits = split_set(3, 21)
    aggs = {"t": {"date_histogram": {"field": "ts", "fixed_interval": "6h"},
                  "aggs": {"ips": {"terms": {"field": "client_ip", "size": 5, "split_size": 1000, "order": {"_key": "asc"}}}}}}
    res = run([img for _, img in splits], MATCH_ALL, DM, max_hits=0, aggs=aggs)
    buckets = res["aggregations"]["t"]["buckets"]
    assert sum(b["doc_count"] for b in buckets) == sum(len(d) for d, _ in splits)
    for b in buckets:
        lo = b["key"] / 1000
        matched = [(docs, [d for d in range(len(docs)) if lo <= docs[d]["ts"] < lo + 6 * 3600]) for docs, _ in splits]
        assert b["ips"] == R.terms_result(R.terms_counts(matched, "client_ip"), 5, "_key", False)


def test_terms_with_missing_field_in_some_splits():
    """a split without the field at all keys its `missing` bucket by address too, so it joins the others"""
    splits = split_set(2, 31)
    bare = [{"log": "alpha", "ts": 1_700_000_000, "status": 1} for _ in range(7)]
    imgs = [img for _, img in splits] + [S.build_split(bare, DM, "ip-bare")]
    res = run(imgs, MATCH_ALL, DM, max_hits=0, aggs=terms_request({"missing": "10.0.0.1", "size": 100}))
    matched = [(docs, range(len(docs))) for docs, _ in splits] + [(bare, range(7))]
    assert res["aggregations"]["ips"] == R.terms_result(R.terms_counts(matched, "client_ip", "10.0.0.1"), 100)
