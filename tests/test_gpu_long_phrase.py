"""Phrases of more than eight tokens on the GPU: QW_NODE_PHRASE through k_phrase_long, checked bit for bit against
the CPU oracle (doc ids, num_hits, f32 scores), and the kernel route of batches that mix short phrases, long phrases
and phrase prefixes."""
import json
import random

import pytest

from quickwit_b200 import ffi, plan as P, service, splitgen as S
from quickwit_b200.proto import DESC
from oracle import oracle as O
from helpers import DOC_ASC, DOC_DESC, SCORE_DESC, assert_same, col_sort, terms_agg
from long_phrase_ref import phrase_ast, values_of, windows
from phrase_prefix_ref import GH_BODY, GH_MAPPING, GH_MSG, gharchive_docs, rewrite_as_phrases
from regex_ref import rewrite_term_sets
from pipeline import search_request

pytestmark = pytest.mark.gpu

MAPPING = {"field_mappings": [{"name": "body", "type": "text", "record": "position", "fieldnorms": True},
                              {"name": "tags", "type": "text", "record": "position"},
                              {"name": "n", "type": "u64", "fast": True}]}
# 11 fixed tokens and an id: the shape of a log line whose template most documents share
TEMPLATE = "INFO org.apache.hadoop.hdfs.server.datanode.DataNode: Receiving block blk_{}"
TEMPLATE_TOKENS = S.tokenize_default(TEMPLATE.format(0))[:11]
SENTENCE = "the quick brown fox jumps over the lazy dog again and again".split()
FILLER = [f"f{i}" for i in range(40)] + ["x", "y", "z", "q", "a", "b"]


def edge_docs(seed, n_filler=12_000, n_template=6_000):
    """Filler text, template lines, and the edge cases: `a b` repeats (counts above 16, driver tf above 32 and 64,
    equally frequent terms), a rare driver with more than 64 positions whose phrase matches only past position 64,
    values of a multi-valued field that a phrase would have to cross, and a sentence in 50 docs."""
    rng = random.Random(seed)
    docs = []
    for i in range(n_filler):
        docs.append({"body": " ".join(rng.choice(FILLER[:40] + ["y", "z"]) for _ in range(rng.randint(3, 30)))})
    for i in range(n_template):
        docs.append({"body": TEMPLATE.format(rng.getrandbits(60))})
    for m in (8, 17, 20, 33, 40, 65, 70, 100, 140):
        docs.append({"body": " ".join(["a", "b"] * m)})
        docs.append({"body": " ".join(["a", "b"] * m + ["a"])})
    tail = "x y z x y z x y z x y z"
    docs.append({"body": "x q " * 70 + tail})
    docs.append({"body": tail + " x q" * 40 + " " + tail + " x q" * 30 + " " + tail})
    docs.append({"body": "x q " * 140})
    for i in range(50):
        docs.append({"body": " ".join(SENTENCE), "tags": ["c d e f g", "h i j k l"] if i % 2 else "c d e f g h i j k l"})
    docs.append({"body": " ".join(SENTENCE[:-1] + ["dog"])})
    rng.shuffle(docs)
    for d, doc in enumerate(docs):
        doc["n"] = d % 50
    return docs


@pytest.fixture(scope="module")
def edge(gpu_ctx):
    img = S.build_split(edge_docs(3), MAPPING, "long-edge")
    gpu_ctx.register_split(img)
    yield img
    gpu_ctx.unregister_split(img.split_id)


def parity(ctx, imgs, plans, label, batch=48):
    """GPU against the oracle (phrase prefixes and term sets rewritten for it), `batch` plans per call; the results."""
    out = []
    for i in range(0, len(plans), batch):
        ims, ps = imgs[i:i + batch], plans[i:i + batch]
        got = ctx.split_search([im.split_id for im in ims], ps)
        for k, (g, im, p) in enumerate(zip(got, ims, ps)):
            assert_same(g, O.split_search(im, rewrite_as_phrases(rewrite_term_sets(p))), ctx=f"{label} #{i + k}")
        out += got
    return out


def test_gharchive_windows(gpu_ctx):
    docs = gharchive_docs()
    img = S.build_split(docs, GH_MAPPING, "gh-long")
    gpu_ctx.register_split(img)
    dm = json.dumps(GH_MAPPING)
    rng = random.Random(23)
    try:
        for field in (GH_MSG, GH_BODY):
            vocab = sorted({t for d in docs for v in values_of(d, field) for t in S.tokenize_default(v)})
            values = [v for d in docs for v in values_of(d, field) if 12 <= len(S.tokenize_default(v)) <= 60]
            phrases = [w for v in rng.sample(values, min(3, len(values))) for w in windows(S.tokenize_default(v), 9, 40)]
            swapped = []
            for p in phrases:
                q = list(p)
                i = rng.randrange(len(q))
                q[i] = rng.choice([t for t in vocab[:200] if t != q[i]])
                swapped.append(q)
            plans = [service.compile_plan(img, search_request(phrase_ast(field, " ".join(p)), max_hits=1000,
                                                              sort_fields=[("_score", DESC)]), dm)
                     for p in phrases + swapped]
            got = parity(gpu_ctx, [img] * len(plans), plans, field)
            assert sum(1 for g in got[:len(phrases)] if g.num_hits) == len(phrases)  # every window matches its doc
            assert all(g.kernel_mask & ffi.KERNEL_PHRASE_LONG and not g.kernel_mask & ffi.KERNEL_PHRASE
                       for g in got[:len(phrases)])
    finally:
        gpu_ctx.unregister_split(img.split_id)


def test_edge_cases(gpu_ctx, edge):
    img = edge
    ph = lambda toks, **kw: P.phrase(img, "body", toks, **kw)
    cases = {
        "a b x5": ["a", "b"] * 5, "b a x5": ["b", "a"] * 5, "a b x20": ["a", "b"] * 20, "a b a x10": ["a", "b", "a"] * 10,
        "a b x64": ["a", "b"] * 64 + ["a"],
        "tail only": "x y z x y z x y z x".split(), "tail long": "x y z x y z x y z x y z".split(),
        "x q": ["x", "q"] * 6,
        "sentence": SENTENCE, "sentence head": SENTENCE[:9], "last token": SENTENCE[:-1] + ["dog"],
        "last token 2": SENTENCE[:-1] + ["the"], "template": TEMPLATE_TOKENS, "template shifted": TEMPLATE_TOKENS[1:] + ["blk"],
    }
    plans, labels = [], []
    for name, toks in cases.items():
        assert len(toks) > ffi.MAX_PHRASE_TERMS
        for k, sort in ((1000, SCORE_DESC), (10, SCORE_DESC), (100, DOC_ASC)):
            plans.append(P.make_plan(ph(toks), k, sort))
            labels.append(f"{name} k={k}")
    # across the values of a multi-valued field (a position gap between them), and within one
    for toks in ("c d e f g h i j k".split(), "c d e f g h i j k l".split(), "g h i j k l c d e".split()):
        plans.append(P.make_plan(P.phrase(img, "tags", toks), 1000, SCORE_DESC))
        labels.append(" ".join(toks))
    got = parity(gpu_ctx, [img] * len(plans), plans, "edge")
    hits = {lab: g.num_hits for lab, g in zip(labels, got)}
    assert hits["a b x5 k=1000"] == 18 and hits["a b x64 k=1000"] == 8
    assert hits["tail only k=1000"] == 2 and hits["x q k=1000"] == 3
    assert hits["sentence k=1000"] == 50 and hits["last token k=1000"] == 1 and hits["last token 2 k=1000"] == 0
    assert hits["template k=1000"] == 6000 and hits["template shifted k=1000"] == 0
    assert hits["c d e f g h i j k"] == 25


def test_long_phrase_as_a_clause(gpu_ctx, edge):
    img = edge
    tmpl = lambda occ=ffi.OCCUR_MUST: P.phrase(img, "body", TEMPLATE_TOKENS, occur=occ)
    sent = lambda occ=ffi.OCCUR_MUST: P.phrase(img, "body", SENTENCE, occur=occ)
    term = lambda t, occ: P.term(img, "body", t, occur=occ)
    roots = [
        tmpl(),
        P.bool_([term("block", ffi.OCCUR_MUST), sent(ffi.OCCUR_SHOULD)]),
        P.bool_([sent(ffi.OCCUR_SHOULD), term("again", ffi.OCCUR_SHOULD), tmpl(ffi.OCCUR_SHOULD)]),
        P.bool_([term("receiving", ffi.OCCUR_MUST), tmpl(ffi.OCCUR_FILTER), P.range_(img, "n", 5, 40)]),
        P.bool_([term("y", ffi.OCCUR_SHOULD), term("z", ffi.OCCUR_SHOULD), tmpl(ffi.OCCUR_MUST_NOT),
                 P.phrase(img, "body", "x y z x y z x y z x".split(), occur=ffi.OCCUR_MUST_NOT)]),
        P.bool_([sent(ffi.OCCUR_MUST), P.phrase(img, "body", ["quick", "brown"], occur=ffi.OCCUR_MUST)]),
    ]
    plans = []
    for root in roots:
        for k, sort in ((10, SCORE_DESC), (1000, SCORE_DESC), (5000, SCORE_DESC), (100, DOC_ASC), (5000, DOC_DESC),
                        (50, [col_sort(img, "n", ffi.ORDER_DESC), DOC_ASC[0]]), (0, DOC_DESC)):
            plans.append(P.make_plan(root, k, sort))
        plans.append(P.make_plan(root, 0, DOC_DESC, aggs=[terms_agg(img, "n")]))
        plans.append(P.make_plan(root, 20, SCORE_DESC, aggs=[terms_agg(img, "n")]))
    gpu_ctx.set_max_hits(20_000)  # K above 4096: the deep selection path
    try:
        got = parity(gpu_ctx, [img] * len(plans), plans, "clauses", batch=9)
    finally:
        gpu_ctx.set_max_hits(4096)
    assert got[0].num_hits == 6000
    assert any(g.kernel_mask & ffi.KERNEL_DEEP_SELECT for g in got)


def oracle_hits(im, clauses, k, sort):
    """The oracle's num_hits of bool(clauses)."""
    return O.split_search(im, rewrite_as_phrases(rewrite_term_sets(P.make_plan(P.bool_(clauses), k, sort)))).num_hits


def oracle_hits_without_each(im, clauses, k, sort):
    """The oracle's num_hits of bool(clauses) with each clause left out in turn."""
    return [oracle_hits(im, clauses[:j] + clauses[j + 1:], k, sort) for j in range(len(clauses))]


def test_mixed_batch_over_several_splits(gpu_ctx):
    imgs = [S.build_split(edge_docs(40 + i, n_filler=3000 + 500 * i, n_template=2000), MAPPING, f"long-mix-{i}")
            for i in range(3)]
    for im in imgs:
        gpu_ctx.register_split(im)
    try:
        short = lambda im: P.make_plan(P.phrase(im, "body", ["quick", "brown", "fox"]), 100, SCORE_DESC)
        long_ = lambda im: P.make_plan(P.phrase(im, "body", SENTENCE), 100, SCORE_DESC)
        tmpl = lambda im: P.make_plan(P.phrase(im, "body", TEMPLATE_TOKENS, occur=ffi.OCCUR_FILTER), 100, DOC_ASC)
        prefix = lambda im: P.make_plan(P.phrase_prefix(im, "body", ["receiving", "block", "b"], 50), 100, DOC_ASC)
        ab = lambda im: P.make_plan(P.phrase(im, "body", ["a", "b", "a", "b"]), 100, SCORE_DESC)
        ords = lambda im, words: sorted(im.term_ord("body", w) for w in words)
        # two term-set nodes beside a phrase, numbered within the plan, then within the call. Each clause cuts the
        # matches, and the nodes' roles differ (filter, must_not), so a bitmap left empty or read by the other node
        # changes the result.
        tset_clauses = lambda im: [P.phrase(im, "body", ["f1", "f2"]), P.term_set(im, "body", ords(im, ["f3", "f4", "f5", "f6"])),
                                   P.term_set(im, "body", ords(im, ["f7"]), occur=ffi.OCCUR_MUST_NOT)]
        tset = lambda im: P.make_plan(P.bool_(tset_clauses(im)), 100, SCORE_DESC)
        for g in parity(gpu_ctx, imgs * 2, [short(im) for im in imgs] + [ab(im) for im in imgs], "short only"):
            assert g.kernel_mask & ffi.KERNEL_PHRASE and not g.kernel_mask & ffi.KERNEL_PHRASE_LONG
        for g in parity(gpu_ctx, imgs * 2, [long_(im) for im in imgs] + [tmpl(im) for im in imgs], "long only"):
            assert g.kernel_mask & ffi.KERNEL_PHRASE_LONG and not g.kernel_mask & ffi.KERNEL_PHRASE
        mixed_imgs = [imgs[0], imgs[1], imgs[2], imgs[1], imgs[0], imgs[2], imgs[1], imgs[2]]
        mixed = [short(imgs[0]), long_(imgs[1]), prefix(imgs[2]), tset(imgs[1]), tmpl(imgs[0]), ab(imgs[2]), prefix(imgs[1]),
                 tset(imgs[2])]
        pre_passes = ffi.KERNEL_PHRASE | ffi.KERNEL_PHRASE_LONG | ffi.KERNEL_TERM_SET
        got = parity(gpu_ctx, mixed_imgs, mixed, "mixed")
        for g in got:
            assert g.kernel_mask & pre_passes == pre_passes
        for j in (3, 7):  # the term-set plans
            im, g = mixed_imgs[j], got[j]
            assert g.num_hits > 0 and g.num_hits not in oracle_hits_without_each(im, tset_clauses(im), 100, SCORE_DESC)
            swapped = tset_clauses(im)
            swapped[1].occur, swapped[2].occur = ffi.OCCUR_MUST_NOT, ffi.OCCUR_FILTER
            assert g.num_hits != oracle_hits(im, swapped, 100, SCORE_DESC)
        # one plan holding a short phrase, a long phrase, a phrase prefix and a term set, each matching docs that no
        # other clause matches
        for im in imgs:
            clauses = [P.phrase(im, "body", ["a", "b"], occur=ffi.OCCUR_SHOULD),
                       P.phrase(im, "body", SENTENCE, occur=ffi.OCCUR_SHOULD),
                       P.phrase_prefix(im, "body", ["receiving", "block", "b"], 50, occur=ffi.OCCUR_SHOULD),
                       P.term_set(im, "body", ords(im, ["q", "z"]), occur=ffi.OCCUR_SHOULD)]
            (g,) = parity(gpu_ctx, [im], [P.make_plan(P.bool_(clauses), 200, DOC_DESC)], "one plan")
            assert g.kernel_mask & pre_passes == pre_passes
            assert g.num_hits > 2000
            assert all(h < g.num_hits for h in oracle_hits_without_each(im, clauses, 200, DOC_DESC))
    finally:
        for im in imgs:
            gpu_ctx.unregister_split(im.split_id)
