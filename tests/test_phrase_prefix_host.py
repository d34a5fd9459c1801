"""Phrase-prefix queries (`phrase_prefix` QueryAst, full_text mode `bool_prefix`) on the CPU: the host compiler's
expansion and lowering, evaluated by the CPU oracle through plans whose PHRASE_PREFIX nodes are rewritten as ORs of
plain phrases, against the reference's REST goldens and a Python brute force."""
import json
import random

import pytest

from quickwit_b200 import ffi, service, splitgen as S
from quickwit_b200.proto import ASC, DESC
from pipeline import bool_, cpu_root_search as cpu_root_search_plain, search_request, term
from phrase_prefix_ref import (GH_BODY, GH_BOOL_PREFIX_COUNTS, GH_MAPPING, GH_MSG, GH_PHRASE_PREFIX_COUNTS,
                               bool_prefix_ast, compiled_expansions, cpu_root_search, doc_positions, expansions,
                               gharchive_docs, parse_plan, phrase_prefix_ast, phrase_prefix_nodes, scan)


@pytest.fixture(scope="module")
def gh():
    return S.build_split(gharchive_docs(), GH_MAPPING, "gharchive")


def _count(imgs, ast, mapping, **kw):
    kw.setdefault("max_hits", 0)
    return cpu_root_search(imgs, ast, mapping, **kw)["num_hits"]


@pytest.mark.parametrize("field,phrase,max_exp,want", GH_PHRASE_PREFIX_COUNTS)
def test_gharchive_match_phrase_prefix(gh, field, phrase, max_exp, want):
    assert _count([gh], phrase_prefix_ast(field, phrase, max_exp), GH_MAPPING) == want


@pytest.mark.parametrize("text,op,want", GH_BOOL_PREFIX_COUNTS)
def test_gharchive_match_bool_prefix(gh, text, op, want):
    assert _count([gh], bool_prefix_ast(GH_BODY, text, op), GH_MAPPING) == want


def test_gharchive_fix_expands_in_byte_order(gh):
    dm = json.dumps(GH_MAPPING)
    for m, want in ((2, [b"fix", b"fixed"]), (3, [b"fix", b"fixed", b"fixes"])):
        plan = service.compile_plan(gh, search_request(phrase_prefix_ast(GH_MSG, "fix", m)), dm)
        assert compiled_expansions(gh, plan) == want


def test_gharchive_automated_commit_hit_and_tokenizers(gh):
    res = cpu_root_search([gh], phrase_prefix_ast(GH_MSG, "automated comm"), GH_MAPPING, max_hits=10,
                          sort_fields=[("_doc", ASC)])
    docs = gharchive_docs()
    (hit,) = res["partial_hits"]
    assert "automated commit" in docs[hit["doc_id"]][GH_MSG]
    # the raw analyzer keeps the phrase whole: one prefix, no term starts with it
    assert _count([gh], phrase_prefix_ast(GH_MSG, "automated comm", tokenizer="raw"), GH_MAPPING) == 0
    assert _count([gh], phrase_prefix_ast(GH_MSG, "automated comm", tokenizer="default"), GH_MAPPING) == 1
    with pytest.raises(ffi.QwGpuError) as e:
        _count([gh], phrase_prefix_ast(GH_MSG, "automated comm", tokenizer="inexistent_tokenizer"), GH_MAPPING)
    assert e.value.code == ffi.EINVALID_QUERY
    with pytest.raises(ffi.QwGpuError) as e:
        _count([gh], bool_prefix_ast(GH_BODY, "file not ch", tokenizer="inexistent_tokenizer"), GH_MAPPING)
    assert e.value.code == ffi.EINVALID_QUERY
    for name in ("lowercase", "whitespace", "chinese_compatible", "source_code_default"):
        with pytest.raises(ffi.QwGpuError) as e:
            _count([gh], phrase_prefix_ast(GH_MSG, "automated comm", tokenizer=name), GH_MAPPING)
        assert e.value.code == ffi.EUNSUPPORTED


# ---- brute force ---------------------------------------------------------------------------------------
VOCAB = ["a", "al", "alp", "alpha", "alphabet", "alps", "alt", "alto", "altos", "b", "be", "bet", "beta", "bets",
         "betting", "c", "ca", "cat", "cats", "catalog", "d", "do", "dog", "dogs", "dot", "e", "zz"]
BF_MAPPING = {"field_mappings": [{"name": "body", "type": "text", "record": "position"},
                                 {"name": "nopos", "type": "text", "record": "freq"},
                                 {"name": "n", "type": "u64", "fast": True}]}


def _bf_docs(rng, n):
    docs = []
    for d in range(n):
        vals = [" ".join(rng.choice(VOCAB) for _ in range(rng.randint(1, 8))) for _ in range(rng.randint(1, 3))]
        docs.append({"body": vals, "nopos": vals[0], "n": d})
    return docs


@pytest.fixture(scope="module")
def bf():
    rng = random.Random(0x5050)
    docs = _bf_docs(rng, 400)
    return docs, S.build_split(docs, BF_MAPPING, "bf")


def test_random_phrase_prefixes_against_a_brute_force(bf):
    docs, img = bf
    pos = [doc_positions(d["body"]) for d in docs]
    dm = json.dumps(BF_MAPPING)
    rng = random.Random(7)
    for it in range(240):
        ntok = rng.randint(1, 5)
        if rng.random() < 0.8:  # a phrase taken from a doc, so that most queries match something
            toks = S.tokenize_default(" ".join(rng.choice(docs)["body"]))
            s = rng.randint(0, max(0, len(toks) - ntok))
            tokens = toks[s:s + ntok]
        else:
            tokens = [rng.choice(VOCAB) for _ in range(ntok)]
        tokens[-1] = tokens[-1][:rng.randint(1, len(tokens[-1]))]
        m = rng.choice([0, 1, 2, 3, 50, 10_000])
        ast = phrase_prefix_ast("body", " ".join(tokens), m)
        exps = expansions(VOCAB, tokens[-1], m)
        want = scan(pos, tokens, exps)
        res = cpu_root_search([img], ast, BF_MAPPING, max_hits=1000, sort_fields=[("_doc", ASC)])
        assert res["num_hits"] == len(want), (tokens, m)
        assert [h["doc_id"] for h in res["partial_hits"]] == want, (tokens, m)
        present = set(t for p in pos for t in p)
        if exps and all(t in present for t in tokens[:-1]):
            plan = service.compile_plan(img, search_request(ast, max_hits=10), dm)
            vocab_exp = [t.encode() for t in expansions(sorted(present), tokens[-1], m)]
            assert compiled_expansions(img, plan) == vocab_exp, (tokens, m)
            _h, root, _t = parse_plan(plan)
            assert bool(phrase_prefix_nodes(root)) == (len(tokens) > 1)


def test_random_bool_prefixes_against_a_brute_force(bf):
    docs, img = bf
    pos = [doc_positions(d["body"]) for d in docs]
    rng = random.Random(11)
    for it in range(80):
        tokens = [rng.choice(VOCAB) for _ in range(rng.randint(1, 4))]
        tokens[-1] = tokens[-1][:rng.randint(1, len(tokens[-1]))]
        op, m = rng.choice(["Or", "And"]), rng.choice([0, 1, 3, 50])
        if len(tokens) == 1:  # make_query: a single token is a plain term query, not a prefix
            want = [d for d, p in enumerate(pos) if tokens[0] in p]
        else:
            exps = expansions(VOCAB, tokens[-1], m)
            sets = [{d for d, p in enumerate(pos) if t in p} for t in tokens[:-1]]
            sets.append({d for d, p in enumerate(pos) if any(e in p for e in exps)})
            want = sorted(set.intersection(*sets) if op == "And" else set.union(*sets))
        res = cpu_root_search([img], bool_prefix_ast("body", " ".join(tokens), op, m), BF_MAPPING, max_hits=1000,
                              sort_fields=[("_doc", ASC)])
        assert [h["doc_id"] for h in res["partial_hits"]] == want, (tokens, op, m)


def test_expansion_is_per_split():
    # split a holds `alpha` and `alps`, split b `alps` and `alto`: with max_expansions 1, `al` is `alpha` in a and
    # `alps` in b, so the `alps` docs of a do not match while those of b do
    a = S.build_split([{"body": "x alpha"}, {"body": "x alps"}, {"body": "alps x"}], BF_MAPPING, "a")
    b = S.build_split([{"body": "x alps"}, {"body": "x alto"}, {"body": "y alps"}], BF_MAPPING, "b")
    dm = json.dumps(BF_MAPPING)
    for ast in (phrase_prefix_ast("body", "al", 1), phrase_prefix_ast("body", "x al", 1)):
        assert compiled_expansions(a, service.compile_plan(a, search_request(ast), dm)) == [b"alpha"]
        assert compiled_expansions(b, service.compile_plan(b, search_request(ast), dm)) == [b"alps"]
    for phrase, per_split in (("al", ([0], [0, 2])), ("x al", ([0], [0]))):
        ast = phrase_prefix_ast("body", phrase, 1)
        got = [[h["doc_id"] for h in cpu_root_search([s], ast, BF_MAPPING, max_hits=10, sort_fields=[("_doc", ASC)])["partial_hits"]]
               for s in (a, b)]
        assert got == list(per_split)
        merged = cpu_root_search([a, b], ast, BF_MAPPING, max_hits=10)
        assert merged["num_hits"] == sum(map(len, per_split))
        assert sorted((h["split_id"], h["doc_id"]) for h in merged["partial_hits"]) == \
            sorted([("a", d) for d in per_split[0]] + [("b", d) for d in per_split[1]])


def test_errors_and_refusals(bf):
    docs, img = bf
    run = lambda ast, **kw: _count([img], ast, BF_MAPPING, **kw)
    score = dict(max_hits=10, sort_fields=[("_score", DESC)])

    def err(ast, code, text=None, **kw):
        with pytest.raises(ffi.QwGpuError) as e:
            cpu_root_search([img], ast, BF_MAPPING, **kw)
        assert e.value.code == code, e.value.msg
        if text:
            assert text in e.value.msg

    err(phrase_prefix_ast("nopos", "alpha be"), ffi.EINVALID_QUERY,
        "trying to run a phrase prefix query on a field which does not have positions indexed")
    assert run(phrase_prefix_ast("nopos", "be")) > 0  # one token needs no positions
    err(phrase_prefix_ast("n", "12"), ffi.EINVALID_QUERY, "non-text field")
    err(phrase_prefix_ast("missing", "al"), ffi.EINVALID_QUERY, "field does not exist")
    assert run(phrase_prefix_ast("missing", "al", lenient=True)) == 0
    assert run(phrase_prefix_ast("body", "!!")) == 0
    assert run(phrase_prefix_ast("body", "!!", zero_terms_query="all")) == len(docs)
    err(phrase_prefix_ast("body", "a b c d e f g h i"), ffi.EUNSUPPORTED)
    err(phrase_prefix_ast("body", "alpha", tokenizer="nope"), ffi.EINVALID_QUERY, "no tokenizer named `nope`")
    # scoring clauses under _score ranking are refused; filter / must_not and every other sort are served
    err(phrase_prefix_ast("body", "alpha be"), ffi.EUNSUPPORTED, **score)
    err(phrase_prefix_ast("body", "al"), ffi.EUNSUPPORTED, **score)
    err(bool_(should=[term("body", "alpha"), phrase_prefix_ast("body", "be")]), ffi.EUNSUPPORTED, **score)
    err(bool_prefix_ast("body", "alpha be"), ffi.EUNSUPPORTED, **score)
    served = bool_(must=[term("body", "alpha")], filter=[phrase_prefix_ast("body", "alpha be")],
                   must_not=[phrase_prefix_ast("body", "do")])
    got = cpu_root_search([img], served, BF_MAPPING, **score)
    pos = [doc_positions(d["body"]) for d in docs]
    want = set(scan(pos, ["alpha", "be"], expansions(VOCAB, "be", 50))) - set(scan(pos, ["do"], expansions(VOCAB, "do", 50)))
    want &= {d for d, p in enumerate(pos) if "alpha" in p}
    assert got["num_hits"] == len(want)
    # the same scores as the query without the prefix clauses, restricted to the docs they keep
    plain = cpu_root_search_plain([img], term("body", "alpha"), BF_MAPPING, max_hits=1000, sort_fields=[("_score", DESC)])
    sc = {h["doc_id"]: h["sort_value"][1] for h in plain["partial_hits"]}
    assert all(sc[h["doc_id"]] == h["sort_value"][1] for h in got["partial_hits"])
    assert run(phrase_prefix_ast("body", "alpha be"), max_hits=5, sort_fields=[("n", DESC)]) > 0
    # a one-token bool_prefix is a plain term query: scored, no prefix expansion
    one = cpu_root_search([img], bool_prefix_ast("body", "alp"), BF_MAPPING, **score)
    assert one["num_hits"] == sum(1 for p in pos if "alp" in p)
    assert one == cpu_root_search_plain([img], term("body", "alp"), BF_MAPPING, **score)
