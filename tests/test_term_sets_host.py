"""Term sets, wildcards and one-token prefixes on the CPU: which form the compiler gives each set group (the
`filter(bool(should: leaf x E))` form of every plan that fits the window program, TERM_SET / COL_SET nodes where it
would not), the boundaries of that rule, the 65 536-value cap, the unchanged literal and scoring refusals, and the
match sets of both forms against a brute force over the documents (the oracle runs the set nodes rewritten as bools of
their children)."""
import numpy as np
import pytest

from quickwit_b200 import ffi, plan as P, splitgen as S
import phrase_corpora as PC
import term_sets_ref as T

SEL_MAPPING = {"field_mappings": [{"name": "f", "type": "text", "tokenizer": "raw"},
                                  {"name": "g", "type": "text", "tokenizer": "raw"},
                                  {"name": "h", "type": "text", "tokenizer": "raw"},
                                  {"name": "n", "type": "u64", "fast": True}]}
N_SEL = 300


@pytest.fixture(scope="module")
def sel():
    # f: a000..a199 and b000..b099; g: c000..c099; h: x00..x39 and y00..y39; n = 0..299 (one doc each)
    docs = [{"f": f"a{d:03d}" if d < 200 else f"b{d - 200:03d}", "g": f"c{d % 100:03d}", "n": d} for d in range(N_SEL)]
    for d in range(80):
        docs[d]["h"] = f"x{d:02d}" if d < 40 else f"y{d - 40:02d}"
    return S.build_split(docs, SEL_MAPPING, "ts-sel")


@pytest.fixture(scope="module")
def docs():
    return T.corpus_docs()


@pytest.fixture(scope="module")
def img(docs):
    return S.build_split(docs, T.MAPPING, "ts-main")


def _compile(img, ast, **kw):
    return T.compile_plan(img, ast, SEL_MAPPING if img.split_id == "ts-sel" else T.MAPPING, **kw)


def _form(leaves):
    """Today's plan of one set group at the root: filter(bool(should: leaf x E)); one leaf: filter(leaf)."""
    for x in leaves:
        x.occur = ffi.OCCUR_SHOULD if len(leaves) > 1 else ffi.OCCUR_FILTER
    inner = leaves[0] if len(leaves) == 1 else P.Node(ffi.NODE_BOOL, ffi.OCCUR_FILTER, children=leaves)
    return T.node_bytes(P.make_plan(P.Node(ffi.NODE_BOOL, ffi.OCCUR_MUST, children=[inner]), 0))


def _terms_form(img, field, names):
    fid = img.field_names().index(field)
    return _form([P.Node(ffi.NODE_TERM, term_ord=img.term_ord(field, x), field_id=fid,
                         weight=P.bm25_weight(img.doc_freq(img.term_ord(field, x)), img.num_docs)) for x in names])


@pytest.mark.parametrize("e", range(1, 65))
def test_groups_that_fit_keep_the_bool_form(sel, e):
    """term_set, one-token prefix (cut at max_expansions = e) and wildcard groups of E <= 64 terms compile node for
    node to today's form."""
    names = [f"a{k:03d}" for k in range(e)]
    want = _terms_form(sel, "f", names)
    cases = [(T.term_set({"f": names}), want), (T.prefix("f", "a", e), want)]
    wildcards = {1: (T.wildcard("f", "a000"), want), 10: (T.wildcard("f", "a00?"), want),
                 40: (T.wildcard("h", "x*"), _terms_form(sel, "h", [f"x{k:02d}" for k in range(40)])),
                 64: (T.wildcard("f", "a0??"), None)}
    if e in wildcards:
        cases.append(wildcards[e])
    for ast, w in cases:
        p = _compile(sel, ast)
        if w is not None:
            assert T.node_bytes(p) == w, ast
        assert not T.set_nodes(p) or e == 64, ast


def test_column_groups_that_fit_keep_the_bool_form(sel):
    c = sel.column_ord("n")
    for e in (1, 2, 64, 92):
        want = _form([P.Node(ffi.NODE_RANGE, column=c, lo=v, hi=v) for v in range(e)])
        assert T.node_bytes(_compile(sel, T.term_set({"n": list(range(e))}))) == want, e


def test_term_boundary(sel):
    """64 TERM leaves fit; 65 turn the group into one TERM_SET node with its term ords ascending."""
    assert not T.set_nodes(_compile(sel, T.prefix("f", "a", 64)))
    for plan in (_compile(sel, T.prefix("f", "a", 65)), _compile(sel, T.wildcard("f", "a0*"))):
        (s,) = T.set_nodes(plan)
        assert s.kind == ffi.NODE_TERM_SET
        ords = [c.term_ord for c in s.children]
        assert ords == sorted(set(ords)) and all(c.kind == ffi.NODE_TERM for c in s.children)
    # 40 + 24 TERMs fit; 40 + 25 convert the larger group only
    both = {"type": "bool", "must": [T.term_set({"f": [f"a{k:03d}" for k in range(40)]}),
                                     T.term_set({"g": [f"c{k:03d}" for k in range(24)]})]}
    assert not T.set_nodes(_compile(sel, both))
    both["must"][1] = T.term_set({"g": [f"c{k:03d}" for k in range(25)]})
    (s,) = T.set_nodes(_compile(sel, both))
    assert len(s.children) == 40 and s.children[0].term_ord == sel.term_ord("f", "a000")


def test_instruction_boundary(sel):
    """A column group of 92 values is 96 instructions and fits; 93 turn into one COL_SET node."""
    assert not T.set_nodes(_compile(sel, T.term_set({"n": list(range(92))})))
    (s,) = T.set_nodes(_compile(sel, T.term_set({"n": list(range(93))})))
    assert s.kind == ffi.NODE_COL_SET and s.column == sel.column_ord("n")
    assert [(c.kind, c.lo, c.hi, c.column) for c in s.children] == [(ffi.NODE_RANGE, v, v, s.column) for v in range(93)]


def test_largest_group_first_ties_in_query_order(sel):
    x40, y40 = T.wildcard("h", "x*"), T.wildcard("h", "y*")
    for first, second in ((x40, y40), (y40, x40)):
        (s,) = T.set_nodes(_compile(sel, {"type": "bool", "must": [first, second]}))
        assert len(s.children) == 40
        assert s.children[0].term_ord == sel.term_ord("h", "x00" if first is x40 else "y00")
    # the largest group goes first, wherever it sits
    a10 = T.wildcard("f", "a00?")
    (s,) = T.set_nodes(_compile(sel, {"type": "bool", "must": [a10, x40, {"type": "bool", "must": [T.wildcard("f", "b00?")]},
                                                               T.wildcard("f", "a0*")]}))
    assert len(s.children) == 100 and s.children[0].term_ord == sel.term_ord("f", "a000")


def test_several_fields_in_one_term_set(sel):
    """Each field of a term_set is its own group: only the one that makes the plan fit converts."""
    ast = T.term_set({"f": [f"a{k:03d}" for k in range(70)], "g": [f"c{k:03d}" for k in range(5)], "n": [1, 2, 3]})
    (s,) = T.set_nodes(_compile(sel, ast))
    assert s.kind == ffi.NODE_TERM_SET and len(s.children) == 70


def test_absent_duplicate_and_all_missing_values(sel):
    vals = [f"a{k:03d}" for k in range(60)] * 2 + [f"zz{k}" for k in range(10)]
    (s,) = T.set_nodes(_compile(sel, T.term_set({"f": vals})))
    assert len(s.children) == 60
    nums = list(range(50)) * 2 + [10**9 + k for k in range(50)]
    (s,) = T.set_nodes(_compile(sel, T.term_set({"n": nums})))
    assert [c.lo for c in s.children] == sorted(set(nums))   # the compiler keeps values outside the split's range
    # every value missing from the split: match-nothing, whichever form
    miss = _compile(sel, T.term_set({"f": [f"zz{k:03d}" for k in range(100)]}))
    assert not T.set_nodes(miss) and T.oracle_search(sel, miss).num_hits == 0


def test_set_cap():
    img = PC.many_terms_split().img
    with pytest.raises(ffi.QwGpuError) as e:
        T.compile_plan(img, T.wildcard("k", "k*"), {"field_mappings": [{"name": "k", "type": "text", "tokenizer": "raw"}]})
    assert e.value.code == ffi.EUNSUPPORTED and "65537" in e.value.msg and "65536" in e.value.msg
    (s,) = T.set_nodes(T.compile_plan(img, T.term_set({"k": [f"k{j:05d}" for j in range(1, 65537)]}),
                                      {"field_mappings": [{"name": "k", "type": "text", "tokenizer": "raw"}]}))
    assert len(s.children) == 65536


def test_literal_errors_and_scoring_refusals_are_unchanged(sel):
    for vals in (["x"], list(range(100)) + ["x"]):
        with pytest.raises(ffi.QwGpuError) as e:
            _compile(sel, T.term_set({"n": vals}))
        assert e.value.code == ffi.EINVALID_QUERY
    score = [("_score", 1)]
    for ast in (T.term_set({"f": ["a000"]}), T.term_set({"f": [f"a{k:03d}" for k in range(100)]}), T.wildcard("f", "a*")):
        with pytest.raises(ffi.QwGpuError) as e:
            _compile(sel, {"type": "bool", "must": [ast]}, max_hits=10, sort_fields=score)
        assert e.value.code == ffi.EUNSUPPORTED
        # in a filter its score is not read
        _compile(sel, {"type": "bool", "filter": [ast]}, max_hits=10, sort_fields=score)


# ---- match sets against the brute force ------------------------------------------------------------------------------
def _values(docs, field, k, rs):
    """k literals for `field`: values of the docs, values no doc holds, and duplicates."""
    held = sorted({v for d in docs for v in (d.get(field) if isinstance(d.get(field), list) else [d.get(field)])
                   if v is not None}, key=str)
    out = [held[i] for i in rs.integers(0, len(held), size=k // 2)]
    missing = {"raw": lambda j: f"r9{j:03d}", "body": lambda j: f"w9{j}", "u": lambda j: 12 + 7 * j, "i": lambda j: 1000 + j,
               "f": lambda j: 0.125 + j, "b": lambda j: True, "dt": lambda j: T.dt_text(T.DT0 + 5_000_000 + j),
               "fo": lambda j: f"s9{j:03d}", "ipi": lambda j: f"10.9.0.{j % 256}", "ipf": lambda j: f"172.16.0.{j % 256}",
               "mu": lambda j: 1000 + j, "ou": lambda j: 400 + j}[field]
    out += [missing(j) for j in range(k // 4)]
    out += out[: k - len(out)]
    return [repr(v) for v in out] if field == "f" else out   # (JSON has no infinities: f64 literals as text)


FIELDS = ("raw", "body", "u", "i", "f", "b", "dt", "fo", "ipi", "ipf", "mu", "ou")


@pytest.mark.parametrize("field", FIELDS)
@pytest.mark.parametrize("k", (3, 150))
def test_term_set_matches_the_brute_force(docs, img, field, k):
    rs = np.random.default_rng(FIELDS.index(field) * 10 + k)
    vals = _values(docs, field, k, rs)
    if field == "body":
        vals = [str(v).split()[1] if " " in str(v) else v for v in vals] + ["Alpha", "alpha"]
    if field == "dt":
        vals = vals + [T.DT0 + 1000 * int(rs.integers(0, 2000)) for _ in range(5)]   # integer literals (ms)
    plan = _compile(img, T.term_set({field: vals}), max_hits=T.N_DOCS)
    converted = bool(T.set_nodes(plan))
    assert converted == (k > 64), field
    got = T.hit_mask(T.oracle_search(img, plan), T.N_DOCS)
    assert np.array_equal(got, T.brute_term_set(docs, {field: vals})), field


def test_f64_edges(docs, img):
    vals = ["-inf", "inf", "-0.0", "0.0", 0.25, -1.5, 1e300] + [0.125 + j for j in range(100)]
    plan = _compile(img, T.term_set({"f": vals}), max_hits=T.N_DOCS)
    assert T.set_nodes(plan)
    got = T.hit_mask(T.oracle_search(img, plan), T.N_DOCS)
    assert np.array_equal(got, T.brute_term_set(docs, {"f": [float(v) for v in vals]}))


def test_positions_of_a_set(docs, img):
    """Sets as must_not, as should under minimum_should_match, in nested bools and under a cache node."""
    rs = np.random.default_rng(3)
    big = {f: _values(docs, f, 120, rs) for f in ("raw", "u", "ipf")}
    n = T.N_DOCS
    m = {f: T.brute_term_set(docs, {f: v}) for f, v in big.items()}
    everything = np.ones(n, dtype=bool)
    cases = [
        ({"type": "bool", "must_not": [T.term_set({"raw": big["raw"]})]}, ~m["raw"]),
        ({"type": "bool", "should": [T.term_set({"raw": big["raw"]}), T.term_set({"u": big["u"]}),
                                     T.term_set({"ipf": big["ipf"]})], "minimum_should_match": 2},
         (m["raw"].astype(int) + m["u"] + m["ipf"]) >= 2),
        ({"type": "bool", "must": [{"type": "bool", "should": [T.term_set({"u": big["u"]}),
                                                               {"type": "bool", "must_not": [T.term_set({"ipf": big["ipf"]})]}]}]},
         m["u"] | ~m["ipf"]),
        ({"type": "bool", "must": [{"type": "cache", "inner": T.term_set({"raw": big["raw"], "u": big["u"]})}],
          "should": [T.term_set({"u": big["u"]})]}, m["raw"] | m["u"]),
        ({"type": "bool", "filter": [{"type": "cache", "inner": T.term_set({"ipf": big["ipf"]})}],
          "must_not": [T.term_set({"raw": big["raw"]})]}, m["ipf"] & ~m["raw"]),
        ({"type": "bool", "must": [{"type": "match_all"}], "filter": [T.term_set({"u": big["u"]})]}, m["u"] & everything),
    ]
    for ast, want in cases:
        plan = _compile(img, ast, max_hits=n)
        assert T.set_nodes(plan), ast
        assert np.array_equal(T.hit_mask(T.oracle_search(img, plan), n), want), ast


def test_wildcard_and_prefix_over_65_terms(docs, img):
    plan = _compile(img, T.wildcard("raw", "r1*"), max_hits=T.N_DOCS)
    (s,) = T.set_nodes(plan)
    assert len(s.children) > 64
    want = np.array([d["raw"].startswith("r1") for d in docs])
    assert np.array_equal(T.hit_mask(T.oracle_search(img, plan), T.N_DOCS), want)
    # match_bool_prefix: `zzz` (absent) OR the first 100 expansions of `w`
    plan = _compile(img, T.bool_prefix("body", "zzz w", 100), max_hits=T.N_DOCS)
    (s,) = T.set_nodes(plan)
    assert len(s.children) == 100
    held = set(sorted({d["body"].split()[1].lower() for d in docs})[:100])
    want = np.array([d["body"].split()[1].lower() in held for d in docs])
    assert np.array_equal(T.hit_mask(T.oracle_search(img, plan), T.N_DOCS), want)
