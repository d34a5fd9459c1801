"""Regex queries (QueryAst `regex`) on the CPU: the host compiler's expansion of a pattern over a split's term
dictionary (quickwit_b200/csrc/regex.h) against a Python brute force, the tokenizer's automatic `(?i)`, every refusal,
the dictionary walk's prefix skipping, and the reference's REST goldens through the CPU oracle."""
import json
import random
import time

import pytest

from quickwit_b200 import ffi, service, splitgen as S
from quickwit_b200.proto import DESC
from pipeline import bool_, search_request, term
from regex_ref import (GH_MAPPING, GH_REGEX_COUNTS, brute_force, compiled_expansions, cpu_root_search, dictionary,
                       gharchive_docs, parse_plan, regex_ast, term_set_nodes)

RAW_MAPPING = {"field_mappings": [{"name": "f", "type": "text", "tokenizer": "raw"},
                                  {"name": "body", "type": "text"},
                                  {"name": "n", "type": "u64", "fast": True},
                                  {"name": "fast_only", "type": "text", "tokenizer": "raw", "fast": True, "indexed": False},
                                  {"name": "declared", "type": "text"},
                                  {"name": "unindexed", "type": "text", "indexed": False}]}


@pytest.fixture(scope="module")
def gh():
    return S.build_split(gharchive_docs(), GH_MAPPING, "gharchive")


@pytest.mark.parametrize("field,regex,want", GH_REGEX_COUNTS)
def test_gharchive_rest_goldens(gh, field, regex, want):
    assert cpu_root_search([gh], regex_ast(field, regex), GH_MAPPING, max_hits=0)["num_hits"] == want


def test_gharchive_goldens_match_the_brute_force(gh):
    docs = gharchive_docs()
    for field, regex, want in GH_REGEX_COUNTS:
        plan = service.compile_plan(gh, search_request(regex_ast(field, regex)), json.dumps(GH_MAPPING))
        exp = set(compiled_expansions(gh, plan))
        tok = (lambda v: [v]) if field == "repo.name" else S.tokenize_default
        assert sum(any(t.encode() in exp for t in tok(d[field])) for d in docs if field in d) == want


# ---- random dictionaries and patterns against `re.fullmatch` ------------------------------------------------------
ASCII = list("abcdefksKS019-. ") + ["\n"]
LATIN1 = ASCII + list("éÉßÿ")
GREEK = ASCII + list("αβΩωΣσς")
CJK = ASCII + list("中文字")
SPECIAL = ["K", "ſ"]  # KELVIN SIGN, LATIN SMALL LETTER LONG S: the (?i) orbits of k and s
POOLS = {"ascii": ASCII, "latin1": LATIN1 + SPECIAL, "greek": GREEK + SPECIAL, "cjk": CJK + SPECIAL}

PERL = [("\\d", "[0-9]"), ("\\w", "[0-9A-Za-z_]"), ("\\s", "[\\t\\n\\x0b\\f\\r ]"), ("\\D", "[^0-9]"),
        ("\\W", "[^0-9A-Za-z_]"), ("[\\d-]", "[0-9\\-]")]
CLASSES = [("[a-f]", "[a-f]"), ("[^a-c]", "[^a-c]"), ("[[:digit:]]", "[0-9]"), ("[[:alpha:]k]", "[A-Za-zk]"),
           ("[^[:alpha:]]", "[^A-Za-z]"), ("[\\-.]", "[\\-.]"), ("[[ab]c]", "[abc]"), ("[\\x61-\\x{64}]", "[a-d]")]
NON_ASCII_CLASSES = [("[α-ω]", "[α-ω]"), ("[^\\x{3b1}-\\x{3c9}]", "[^α-ω]"), ("[中文]", "[中文]")]
NON_ASCII_LITERALS = ["é", "ß", "α", "Σ", "中", "K", "ſ"]


def gen(rng, depth, ci, names):
    """(pattern for the product, the same pattern for Python's re) over the served subset; ci: under (?i)."""
    r = rng.random()
    if depth <= 0 or r < 0.3:
        k = rng.random()
        if k < 0.35:
            c = rng.choice("abcdefksKS019-")
            return c, c
        if k < 0.45 and not ci:
            c = rng.choice(NON_ASCII_LITERALS)
            return c, c
        if k < 0.55:
            c = rng.choice(".-")
            return "\\" + c, "\\" + c
        if k < 0.65:
            return ".", "."
        if k < 0.75:
            return rng.choice(PERL)
        pool = CLASSES + ([] if ci else NON_ASCII_CLASSES)
        return rng.choice(pool)
    if r < 0.5:
        parts = [gen(rng, depth - 1, ci, names) for _ in range(rng.randint(2, 3))]
        return "".join(p for p, _ in parts), "".join(q for _, q in parts)
    if r < 0.6:
        parts = [gen(rng, depth - 1, ci, names) for _ in range(rng.randint(2, 3))]
        return "|".join(p for p, _ in parts), "|".join(q for _, q in parts)
    if r < 0.8:
        a, b = gen(rng, depth - 1, ci, names)
        op = rng.choice(["*", "+", "?", "{2}", "{1,}", "{0,2}", "{1,3}"])
        return "(?:" + a + ")" + op, "(?:" + b + ")" + op
    if r < 0.9:
        flag = rng.choice(["i", "s", "-i"])
        inner_ci = (ci or flag == "i") and flag != "-i"
        a, b = gen(rng, depth - 1, inner_ci, names)
        return "(?" + flag + ":" + a + ")", "(?" + flag + ":" + b + ")"
    a, b = gen(rng, depth - 1, ci, names)
    if rng.random() < 0.5:
        return "(" + a + ")", "(" + b + ")"
    names.append(f"g{len(names)}")
    return f"(?P<{names[-1]}>" + a + ")", f"(?P<{names[-1]}>" + b + ")"


def random_split(rng, pool, n_terms):
    terms = {"".join(rng.choice(pool) for _ in range(rng.randint(1, 5))) for _ in range(n_terms)}
    return S.build_split([{"f": t} for t in sorted(terms)], RAW_MAPPING, "rnd")


@pytest.mark.parametrize("flavor", sorted(POOLS))
def test_random_patterns_match_the_brute_force(flavor):
    rng = random.Random(0x5EED + sorted(POOLS).index(flavor))
    served = refused = 0
    for _ in range(6):
        img = random_split(rng, POOLS[flavor], 250)
        non_ascii = any(max(b) >= 0x80 for _t, b in dictionary(img, "f"))
        for _ in range(40):
            ci = rng.random() < 0.3
            ours, py = gen(rng, 3, ci, [])
            if ci:
                ours, py = "(?i)" + ours, "(?i)" + py
            try:
                ords, _steps = service.regex_terms(img, "f", ours)
            except ffi.QwGpuError as e:
                # only the Perl classes may refuse a split, and only one with a non-ASCII term
                assert e.code == ffi.EUNSUPPORTED and "Perl classes" in str(e), (ours, e)
                assert non_ascii and any(p in ours for p, _ in PERL), ours
                refused += 1
                continue
            got = [b for t, b in dictionary(img, "f") if t in set(ords)]
            assert got == brute_force(img, "f", py), (ours, py)
            served += 1
    assert served > 150
    if flavor == "ascii":
        assert refused == 0


def test_case_folding_orbits():
    img = S.build_split([{"f": t} for t in ["k", "K", "K", "s", "S", "ſ", "x", "Kx", "ks"]], RAW_MAPPING, "fold")
    words = lambda ords: sorted(b.decode() for t, b in dictionary(img, "f") if t in set(ords))
    run = lambda re_: words(service.regex_terms(img, "f", re_)[0])
    assert run("(?i)k") == sorted(["k", "K", "K"])
    assert run("(?i)S") == sorted(["s", "S", "ſ"])
    assert run("(?i)[j-l]") == sorted(["k", "K", "K"])
    assert run("(?i)[^k]") == sorted(["s", "S", "ſ", "x"])
    assert run("k") == ["k"]
    assert run("(?i)(?-i:k)") == ["k"]
    assert run("(?i)kx") == ["Kx"]
    for bad in ("(?i)é", "(?i)[α-ω]", "(?i)\\x{212a}"):
        with pytest.raises(ffi.QwGpuError) as e:
            service.regex_terms(img, "f", bad)
        assert e.value.code == ffi.EUNSUPPORTED


# ---- the tokenizer's automatic (?i) -------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def cased():
    docs = [{"f": v, "body": v} for v in ["ABC", "abc", "Abc", "xyz"]]
    return S.build_split(docs, RAW_MAPPING, "cased")


def _expand(img, field, regex):
    plan = service.compile_plan(img, search_request(regex_ast(field, regex)), json.dumps(RAW_MAPPING))
    return compiled_expansions(img, plan)


def test_auto_case_insensitive_rule(cased):
    # raw: the pattern as given
    assert _expand(cased, "f", "ABC") == [b"ABC"]
    assert _expand(cased, "f", "abc") == [b"abc"]
    assert _expand(cased, "f", "(?i)abc") == [b"ABC", b"Abc", b"abc"]
    # default (lowercasing) tokenizer: the terms are lowercase, the pattern gains (?i)
    assert _expand(cased, "body", "ABC") == [b"abc"]
    assert _expand(cased, "body", "A.C") == [b"abc"]
    # ... unless the text up to the first `)` of a leading `(?` holds an `i` — `(?-i)` included
    assert _expand(cased, "body", "(?-i)ABC") == []
    assert _expand(cased, "body", "(?-i)abc") == [b"abc"]
    assert _expand(cased, "body", "(?i)ABC") == [b"abc"]
    assert _expand(cased, "body", "(?s)ABC") == [b"abc"]
    assert _expand(cased, "body", "(?P<id>ABC)") == []  # the string test sees the `i` of `id`


# ---- refusals -----------------------------------------------------------------------------------------------------
INVALID = ["(abc", "abc)", "[abc", "[z-a]", "*a", "a|*", "x{3,1}", "x{a}", "x{2", "\\", "\\q", "(?z)a", "(?)a", "(?-)a",
           "(?ii)a", "a(?=b)", "a(?!b)", "(?<=a)b", "(?<!a)b", "(a)\\1", "(?P=n)", "^abc", "abc$", "\\Aabc", "abc\\z",
           "a\\bc", "a\\Bc", "[[:foo:]]", "(?P<1n>a)", "(?P<n>a)(?P<n>b)", "\\x{110000}", "\\xZ1", "[\\d-z]"]
UNSUPPORTED = ["a*?", "a+?", "a??", "a{1,2}?", "(?U)a*", "\\p{L}", "\\PL", "(?-u)a", "(?x)a b", "a**", "[a&&b]",
               "[a--b]", "[a~~b]", "x{,3}", "\\u0041", "\\/", "(?R)a"]


@pytest.mark.parametrize("pattern", INVALID)
def test_invalid_patterns_fail_to_parse(cased, pattern):
    with pytest.raises(ffi.QwGpuError) as e:
        _expand(cased, "f", pattern)
    assert e.value.code == ffi.EINVALID_QUERY and "failed to parse regex" in str(e.value), (pattern, e.value)


@pytest.mark.parametrize("pattern", UNSUPPORTED)
def test_unsupported_patterns_are_refused(cased, pattern):
    with pytest.raises(ffi.QwGpuError) as e:
        _expand(cased, "f", pattern)
    assert e.value.code == ffi.EUNSUPPORTED, (pattern, e.value)


def test_served_syntax(cased):
    for p in ["(?P<a>A)BC", "(?<a>A)BC", "(?:A)BC", "A(?i:b)C", "(?i)a(?-i)BC", "[A]B\\x43", "A\\x{42}C", "ABC{1}",
              "A[[:upper:]]{2}", "(?m)ABC", "(?u)ABC", "(?is)abc", "(?i-s:abc)", "A(B|X)C", "ABC|xyz|", "[]A]BC"]:
        assert b"ABC" in _expand(cased, "f", p), p


def test_field_resolution(cased):
    dm = json.dumps(RAW_MAPPING)
    run = lambda field: service.compile_plan(cased, search_request(regex_ast(field, "a.*")), dm)
    for field, msg in (("missing", "field does not exist"), ("n", "non-text field"), ("fast_only", "not full-text searchable"),
                       ("unindexed", "not full-text searchable")):
        with pytest.raises(ffi.QwGpuError) as e:
            run(field)
        assert e.value.code == ffi.EINVALID_QUERY and msg in str(e.value), field
    # declared, but without a term in this split: matches nothing, and the pattern is still checked
    assert parse_plan(run("declared"))[1].kind == ffi.NODE_NONE
    with pytest.raises(ffi.QwGpuError) as e:
        service.compile_plan(cased, search_request(regex_ast("declared", "(a")), dm)
    assert e.value.code == ffi.EINVALID_QUERY


def test_perl_class_refused_only_where_the_walk_meets_non_ascii():
    ascii_img = S.build_split([{"f": t} for t in ["a1", "b22", "zz", "a-"]], RAW_MAPPING, "a")
    mixed = S.build_split([{"f": t} for t in ["a1", "b22", "zz", "aé", "é1"]], RAW_MAPPING, "m")
    assert len(service.regex_terms(ascii_img, "f", "a\\d")[0]) == 1
    # the walk tests \d only after an `a`: `é1` dies at `é` against the literal, `aé` meets \d with é
    with pytest.raises(ffi.QwGpuError) as e:
        service.regex_terms(mixed, "f", "a\\d")
    assert e.value.code == ffi.EUNSUPPORTED and "Perl classes" in str(e.value)
    # a walk that never tests the class against a non-ASCII code point is served
    assert len(service.regex_terms(mixed, "f", "b\\d+")[0]) == 1


def test_repetitions_of_the_empty_string_compile_at_once(cased):
    """A body that can only match the empty string (`a{0}`, or an alternation / group of such) adds no state, so the
    state bound cannot end its repetition: the compiler drops it whole instead of expanding the count."""
    t = time.perf_counter()
    for p in ("x(?:a{0}){400000000}", "x(?:(?:a{0}){100000}){100000}", "x(?:(?:(?:a{0}|(?:b){0}){100000}){100000}){100000}",
              "x(?:a{0}|){4000000000}", "x(?:a{0})+"):
        assert _expand(cased, "f", p) == [], p  # through the compiler: no term is just `x`
        assert service.regex_terms(cased, "f", p + "yz")[0] == [t_ for t_, b in dictionary(cased, "f") if b == b"xyz"], p
    assert time.perf_counter() - t < 2.0
    # a body that consumes adds a state per copy: the bound ends the count
    for p in ("(?:a{0}b){20000}", "(?:(?:a{0}b){100000}){100000}"):
        with pytest.raises(ffi.QwGpuError) as e:
            _expand(cased, "f", p)
        assert e.value.code == ffi.EUNSUPPORTED and "states" in str(e.value), p


def test_automaton_state_bound_of_the_walk():
    """`.*a.{16}` needs an automaton state per pattern of `a`s in the last 17 characters: a walk over 100 000 random
    terms of 20 letters builds more than 65 536 of them and is refused; `.*a.{3}` over the same terms is served."""
    rng = random.Random(7)
    text = " ".join("".join(rng.choice("ab") for _ in range(20)) for _ in range(100_000))
    img = S.build_split([{"body": text}], RAW_MAPPING, "ab")
    with pytest.raises(ffi.QwGpuError) as e:
        service.regex_terms(img, "body", ".*a.{16}")
    assert e.value.code == ffi.EUNSUPPORTED and "automaton states" in str(e.value)
    words = [b.decode() for _t, b in dictionary(img, "body")]
    ords, _ = service.regex_terms(img, "body", ".*a.{3}")
    assert len(ords) == sum(w[-4] == "a" for w in words)


def test_state_bound_both_sides(cased):
    assert _expand(cased, "f", "x{9999}") == []  # 10 000 states with the final one: served (matches nothing here)
    for p in ("x{10000}", "x{5000}y{5000}", "(?:a|b){5000}"):
        with pytest.raises(ffi.QwGpuError) as e:
            _expand(cased, "f", p)
        assert e.value.code == ffi.EUNSUPPORTED and "states" in str(e.value), p


# ---- expansion limit and scoring position ---------------------------------------------------------------------------

@pytest.fixture(scope="module")
def wide():
    """One doc holding a00000 .. a65535 (65 536 terms) and b0."""
    text = " ".join(f"a{i:05d}" for i in range(ffi.MAX_SET_TERMS)) + " b0"
    return S.build_split([{"body": text, "n": 1}, {"body": "c1", "n": 2}], RAW_MAPPING, "wide")


def test_expansion_limit(wide):
    dm = json.dumps(RAW_MAPPING)
    plan = service.compile_plan(wide, search_request(regex_ast("body", "a.*")), dm)
    (node,) = term_set_nodes(parse_plan(plan)[1])
    assert len(node.children) == ffi.MAX_SET_TERMS
    with pytest.raises(ffi.QwGpuError) as e:
        service.compile_plan(wide, search_request(regex_ast("body", "[ab].*")), dm)
    assert e.value.code == ffi.EUNSUPPORTED and str(ffi.MAX_SET_TERMS) in str(e.value)


def test_scoring_position_under_score_ranking(cased):
    dm = json.dumps(RAW_MAPPING)
    score = [("_score", DESC)]
    for ast in (regex_ast("f", "A.*"), bool_(must=[regex_ast("f", "A.*"), term("body", "abc")]),
                bool_(should=[regex_ast("f", "A.*"), term("body", "abc")])):
        with pytest.raises(ffi.QwGpuError) as e:
            service.compile_plan(cased, search_request(ast, max_hits=10, sort_fields=score), dm)
        assert e.value.code == ffi.EUNSUPPORTED and "regex" in str(e.value)
    for ast, want in ((bool_(must=[term("body", "abc")], filter=[regex_ast("f", "A.*")]), 2),
                      (bool_(must=[term("body", "abc")], must_not=[regex_ast("f", "a.*")]), 2)):
        plan = service.compile_plan(cased, search_request(ast, max_hits=10, sort_fields=score), dm)
        assert len(term_set_nodes(parse_plan(plan)[1])) == 1
        res = cpu_root_search([cased], ast, RAW_MAPPING, max_hits=10, sort_fields=score)
        assert res["num_hits"] == want
    # the same regex in a scoring position is served when the sort does not read scores
    assert cpu_root_search([cased], regex_ast("f", "A.*"), RAW_MAPPING, max_hits=10)["num_hits"] == 2


# ---- the dictionary walk skips dead prefixes ------------------------------------------------------------------------

def test_walk_resumes_and_skips_dead_prefixes():
    """Counted automaton transitions (host code: a count, not a time). 200 000 terms x000000 .. x199999 plus 100 terms
    apieu00 .. apieu99: an anchored literal costs O(matches x length + log N), a pattern that can die nowhere touches
    every term once past the shared prefixes."""
    n = 200_000
    text = " ".join(f"x{i:06d}" for i in range(n)) + " " + " ".join(f"apieu{i:02d}" for i in range(100))
    img = S.build_split([{"body": text}], RAW_MAPPING, "big")
    ords, steps = service.regex_terms(img, "body", "apieu.*")
    assert len(ords) == 100
    assert steps < 100 * 3 + 64, steps  # 5 shared bytes once, then 2 per term, plus the dying probe of `x`
    ords, steps = service.regex_terms(img, "body", "x1.*")
    assert len(ords) == 100_000 and steps < 3 * 100_000, steps  # resumes at the common prefix: about 1.1 per term
    ords, steps = service.regex_terms(img, "body", "q.*")
    assert ords == [] and steps <= 3
    _ords, steps = service.regex_terms(img, "body", ".*9")
    assert steps > n  # nothing dies: every term is walked (from its common prefix with the one before)
