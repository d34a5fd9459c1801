"""Phrases of more than eight tokens on the CPU: the host compiler's plan (one QW_NODE_PHRASE of up to
QW_MAX_PHRASE_LEN TERM children), its refusals, and the CPU oracle's matches and phrase counts against
scoring_ref.phrase_counts on a random corpus and on the gharchive fixture."""
import json
import random

import numpy as np
import pytest

from quickwit_b200 import ffi, service, splitgen as S
from quickwit_b200.proto import DESC
from oracle import oracle as O
from long_phrase_ref import TokenPostings, expected_scores, phrase_ast, phrase_weight, values_of, windows
from phrase_prefix_ref import GH_BODY, GH_MAPPING, GH_MSG, gharchive_docs, parse_plan
from pipeline import search_request
from scoring_ref import phrase_counts

MAPPING = {"field_mappings": [{"name": "body", "type": "text", "record": "position", "fieldnorms": True},
                              {"name": "nopos", "type": "text", "record": "freq"},
                              {"name": "n", "type": "u64", "fast": True}]}
VOCAB = [f"w{i}" for i in range(300)]


def random_docs(seed, n=600):
    """Values that are either a run of the sequence w0 w1 w2 ... (long phrases match) or draws from a dozen words
    (short repeats), one to three values per doc; doc 0 holds the whole vocabulary."""
    rng = random.Random(seed)
    docs = [{"body": " ".join(VOCAB), "nopos": " ".join(VOCAB), "n": 0}]
    for d in range(1, n):
        vals = []
        for _ in range(rng.randint(1, 3)):
            k = rng.randint(1, 60)
            if rng.random() < 0.5:
                s = rng.randint(0, 40)
                vals.append(" ".join(VOCAB[s:s + k]))
            else:
                vals.append(" ".join(rng.choice(VOCAB[:12]) for _ in range(k)))
        docs.append({"body": vals, "nopos": vals[0], "n": d})
    for j in range(3):  # `w0 w1 w0 w1 ...`: phrase counts above the tf-factor table's 16 rows
        alt = " ".join(VOCAB[i % 2] for i in range(40 + 30 * j))
        docs.append({"body": alt, "nopos": alt, "n": len(docs)})
    return docs


@pytest.fixture(scope="module")
def rnd():
    docs = random_docs(0x10F)
    return docs, S.build_split(docs, MAPPING, "long-rnd")


@pytest.fixture(scope="module")
def gh():
    docs = gharchive_docs()
    return docs, S.build_split(docs, GH_MAPPING, "gharchive")


def compile_(img, ast, mapping, **kw):
    return service.compile_plan(img, search_request(ast, **kw), json.dumps(mapping))


def phrase_nodes(plan):
    _h, root, _t = parse_plan(plan)
    out, stack = [], [root]
    while stack:
        n = stack.pop()
        if n.kind == ffi.NODE_PHRASE:
            out.append(n)
        else:
            stack.extend(n.children)
    return out


def numpy_weight(img, field, tokens):
    """(sum of the terms' f32 idf in phrase order, duplicates included) * (1 + k1), in numpy."""
    f32 = np.float32
    s = f32(0)
    for t in tokens:
        df = img.doc_freq(img.term_ord(field, t))
        s = f32(s + np.log(f32(1) + (f32(img.num_docs - df) + f32(0.5)) / (f32(df) + f32(0.5)), dtype=np.float32))
    return f32(s * f32(2.2))


@pytest.mark.parametrize("n", [9, 16, 64, 256])
def test_compiled_plan(rnd, n):
    _docs, img = rnd
    for tokens in (VOCAB[:n], [VOCAB[(i * 5) % 7] for i in range(n)], VOCAB[300 - n:]):
        for mode in ("phrase", "phrase_fallback_to_intersection"):
            (node,) = phrase_nodes(compile_(img, phrase_ast("body", " ".join(tokens), mode), MAPPING, max_hits=10))
            assert len(node.children) == n
            assert [c.kind for c in node.children] == [ffi.NODE_TERM] * n
            assert [c.lo for c in node.children] == list(range(n))
            assert [c.term_ord for c in node.children] == [img.term_ord("body", t) for t in tokens]
            assert np.float32(node.weight) == phrase_weight(img, "body", tokens)
            ref = numpy_weight(img, "body", tokens)
            assert abs(float(node.weight) - float(ref)) <= 1e-6 * float(ref), (n, tokens[:3])


def test_refusals_and_match_none(rnd):
    docs, img = rnd

    def err(ast, code):
        with pytest.raises(ffi.QwGpuError) as e:
            compile_(img, ast, MAPPING, max_hits=10)
        assert e.value.code == code, e.value.msg
        return e.value.msg

    msg = err(phrase_ast("body", " ".join(VOCAB[:257])), ffi.EUNSUPPORTED)
    assert "256" in msg
    assert "256" in err(phrase_ast("body", " ".join(VOCAB[:257]), "phrase_fallback_to_intersection"), ffi.EUNSUPPORTED)
    assert phrase_nodes(compile_(img, phrase_ast("body", " ".join(VOCAB[:256])), MAPPING, max_hits=10))
    # a token missing from the split: match_none
    for tokens in (VOCAB[:12] + ["absent"], ["absent"] + VOCAB[:40]):
        plan = compile_(img, phrase_ast("body", " ".join(tokens)), MAPPING, max_hits=10)
        assert not phrase_nodes(plan)
        assert O.split_search(img, plan).num_hits == 0
    # a field without positions: phrase mode is an invalid query, the fallback mode an intersection of terms
    err(phrase_ast("nopos", " ".join(VOCAB[:20])), ffi.EINVALID_QUERY)
    plan = compile_(img, phrase_ast("nopos", " ".join(VOCAB[:20]), "phrase_fallback_to_intersection"), MAPPING, max_hits=10)
    assert not phrase_nodes(plan)
    want = sum(1 for d in docs if set(VOCAB[:20]) <= set(S.tokenize_default(d["nopos"])))
    assert O.split_search(img, plan).num_hits == want > 0


def check_counts(img, tp, field, mapping, phrases, fieldnorms):
    """The oracle's hits of each phrase under _score ranking, against phrase_counts and the f32 score of its count.
    Returns the number of phrases that matched something and the largest phrase count seen."""
    matched, top = 0, 0
    for tokens in phrases:
        plan = compile_(img, phrase_ast(field, " ".join(tokens)), mapping, max_hits=img.num_docs,
                        sort_fields=[("_score", DESC)])
        got = O.split_search(img, plan)
        if any((field, t) not in tp.postings for t in tokens):
            assert got.num_hits == 0
            continue
        docs, counts = phrase_counts(tp, field, tokens)
        assert got.num_hits == len(docs), tokens
        by_doc = {h[0]: h[4] for h in got.hits}
        assert sorted(by_doc) == docs.tolist(), tokens
        if len(docs):
            (node,) = phrase_nodes(plan)
            want = expected_scores(img, field, counts, docs, tp.lengths, node.weight, fieldnorms)
            have = np.array([by_doc[int(d)] for d in docs], dtype=np.float32)
            assert np.array_equal(have.view(np.uint32), want.view(np.uint32)), tokens
            matched += 1
            top = max(top, int(counts.max()))
    return matched, top


def swapped(rng, tokens, pool, at=None):
    out = list(tokens)
    i = rng.randrange(len(out)) if at is None else at
    out[i] = rng.choice([t for t in pool if t != out[i]])
    return out


def test_oracle_counts_on_a_random_corpus(rnd):
    docs, img = rnd
    tp = TokenPostings(docs, "body")
    rng = random.Random(5)
    pool = VOCAB[:60]
    phrases = []
    for _ in range(40):
        toks = S.tokenize_default(rng.choice(values_of(rng.choice(docs[1:]), "body")))
        if len(toks) >= 9:
            w = windows(toks, 9, min(40, len(toks)))
            phrases += rng.sample(w, min(4, len(w)))
    phrases += [swapped(rng, p, pool) for p in phrases[:40]] + [swapped(rng, p, pool, len(p) - 1) for p in phrases[:40]]
    # repeated tokens: counts above the tf-factor table's 16 rows need a doc of many repeats
    phrases += [[VOCAB[i % 2] for i in range(10)], [VOCAB[i % 3] for i in range(9)], VOCAB[:9], VOCAB[30:70]]
    matched, top = check_counts(img, tp, "body", MAPPING, phrases, fieldnorms=True)
    assert matched > 60 and top > 16


def test_oracle_counts_on_gharchive(gh):
    docs, img = gh
    rng = random.Random(17)
    for field in (GH_MSG, GH_BODY):
        tp = TokenPostings(docs, field)
        values = [v for d in docs for v in values_of(d, field) if len(S.tokenize_default(v)) >= 12]
        pool = sorted({t for (_f, t) in tp.postings})
        phrases = []
        for v in rng.sample(values, min(6, len(values))):
            w = windows(S.tokenize_default(v), 9, 40)
            phrases += rng.sample(w, min(12, len(w)))
        cut = len(phrases)  # every window cut from a value matches at least its own doc
        phrases += [swapped(rng, p, pool) for p in phrases[:20]] + [swapped(rng, p, pool, len(p) - 1) for p in phrases[:20]]
        matched, _top = check_counts(img, tp, field, GH_MAPPING, phrases, fieldnorms=False)
        assert matched >= cut >= 30, field
