"""Phrase-prefix queries on the GPU: QW_NODE_PHRASE_PREFIX through k_phrase's suffix stage, checked bit for bit
against the CPU oracle (which evaluates the same plan rewritten as an OR of plain phrases), against the GPU's own
OR-of-phrases plan, and against the reference's REST goldens through the full request path."""
import json
import random

import pytest

from quickwit_b200 import ffi, plan as P, proto, service, splitgen as S
from quickwit_b200.proto import ASC, DESC
from oracle import oracle as O
from helpers import DOC_ASC, DOC_DESC, SCORE_DESC, assert_same, col_sort, terms_agg
from pipeline import bool_, leafify, search_request, term
from phrase_prefix_ref import (GH_BODY, GH_BOOL_PREFIX_COUNTS, GH_MAPPING, GH_PHRASE_PREFIX_COUNTS, bool_prefix_ast,
                               cpu_root_search, gharchive_docs, phrase_prefix_ast, rewrite_as_phrases)

pytestmark = pytest.mark.gpu

# prefix-sharing words: `al*`, `be*`, `ga*` expand to several terms of very different frequencies
_VOCAB = ["alpha", "alps", "alt", "alto", "altos", "beta", "bet", "bets", "betting", "gamma", "gam", "game", "games",
          "delta", "eta", "zeta", "theta", "iota"]
_WEIGHTS = [12, 3, 2, 1, 0.2, 10, 4, 1, 0.1, 8, 2, 1, 0.5, 6, 5, 4, 3, 0.05]
MAPPING = {"field_mappings": [{"name": "body", "type": "text", "record": "position", "fieldnorms": True},
                              {"name": "tags", "type": "text", "record": "position"},
                              {"name": "n", "type": "u64", "fast": True}]}


def _docs(n, seed):
    rnd = random.Random(seed)
    docs = []
    for i in range(n):
        doc = {"body": " ".join(rnd.choices(_VOCAB, _WEIGHTS, k=3 + (i * 37) % 38)), "n": i % 50}
        if i % 3 == 0:
            doc["tags"] = [" ".join(rnd.choices(_VOCAB[:9], k=1 + i % 3)) for _ in range(1 + i % 4)]
        docs.append(doc)
    return docs


@pytest.fixture(scope="module")
def pp_split(gpu_ctx):
    img = S.build_split(_docs(20_000, 11), MAPPING, "prefix-0")
    gpu_ctx.register_split(img)
    yield img
    gpu_ctx.unregister_split(img.split_id)


def run_both(sctx, img, plan, **kw):
    got = sctx.split_search([img.split_id], [plan])[0]
    want = O.split_search(img, rewrite_as_phrases(plan))
    assert_same(got, want, **kw)
    return got


def or_plan(img, field, tokens, m, occur=ffi.OCCUR_MUST):
    node = P.phrase_prefix(img, field, tokens, m, occur=occur)
    return P.phrase_prefix_as_phrases(node) if node.kind == ffi.NODE_PHRASE_PREFIX else node


CASES = [(["alpha", "be"], 50), (["beta", "al"], 50), (["alpha", "alpha", "al"], 3), (["gamma", "be"], 1),
         (["iota", "a"], 50), (["alpha", "beta", "gamma", "d"], 50), (["eta", "z"], 50), (["alps", "b"], 2),
         (["theta", "zeta", "eta", "delta", "gamma", "beta", "a"], 50), (["beta", "x"], 50)]


def test_phrase_prefixes_against_the_oracle(gpu_ctx, pp_split):
    img = pp_split
    n_hits = []
    for tokens, m in CASES:
        node = P.phrase_prefix(img, "body", tokens, m)
        for k, sort in ((0, DOC_DESC), (10, DOC_ASC), (1000, DOC_DESC), (10, [col_sort(img, "n", ffi.ORDER_ASC)])):
            got = run_both(gpu_ctx, img, P.make_plan(node, k, sort), ctx=f"{tokens} m={m} k={k}")
            if node.kind == ffi.NODE_PHRASE_PREFIX:
                assert got.kernel_mask & ffi.KERNEL_PHRASE
        # the same results as the OR of one plain phrase per expansion, on the GPU
        got, cross = gpu_ctx.split_search([img.split_id] * 2, [P.make_plan(node, 1000, DOC_ASC),
                                                               P.make_plan(or_plan(img, "body", tokens, m), 1000, DOC_ASC)])
        assert (cross.num_hits, cross.hits) == (got.num_hits, got.hits), tokens
        n_hits.append(got.num_hits)
    assert max(n_hits) > 3000 and 0 < min(x for x in n_hits if x) < 300 and 0 in n_hits
    for tokens in (["alpha", "be"], ["beta", "beta", "al"]):  # multi-valued field without fieldnorms
        run_both(gpu_ctx, img, P.make_plan(P.phrase_prefix(img, "tags", tokens, 50), 50, DOC_ASC), ctx=f"tags {tokens}")


def test_phrase_prefixes_as_clauses(gpu_ctx, pp_split):
    img = pp_split
    pp = lambda tokens, occ, m=50: P.phrase_prefix(img, "body", tokens, m, occur=occ)
    t = lambda name, occ: P.term(img, "body", name, occur=occ)
    scored = [  # scored terms under _score ranking, the phrase prefix where its score is not read
        P.bool_([t("gamma", ffi.OCCUR_MUST), pp(["alpha", "be"], ffi.OCCUR_FILTER)]),
        P.bool_([t("gamma", ffi.OCCUR_SHOULD), t("delta", ffi.OCCUR_SHOULD), pp(["beta", "al"], ffi.OCCUR_MUST_NOT)]),
        P.bool_([P.phrase(img, "body", ["alpha", "beta"]), pp(["gamma", "ga"], ffi.OCCUR_FILTER), P.range_(img, "n", 5, 40)]),
    ]
    for i, root in enumerate(scored):
        for k in (0, 10, 1000):
            run_both(gpu_ctx, img, P.make_plan(root, k, SCORE_DESC), ctx=f"scored {i} k={k}")
    unscored = [
        P.bool_([pp(["alpha", "be"], ffi.OCCUR_MUST), t("eta", ffi.OCCUR_SHOULD), pp(["gamma", "al"], ffi.OCCUR_MUST_NOT)]),
        P.bool_([pp(["alpha", "be"], ffi.OCCUR_SHOULD), pp(["delta", "ga"], ffi.OCCUR_SHOULD), t("iota", ffi.OCCUR_SHOULD)],
                min_should_match=2),
        P.bool_([pp(["eta", "a"], ffi.OCCUR_SHOULD, 1), P.phrase(img, "body", ["zeta", "eta"], occur=ffi.OCCUR_SHOULD)]),
        P.bool_([pp(["alpha", "be"], ffi.OCCUR_MUST), pp(["alpha"], ffi.OCCUR_FILTER)]),
    ]
    for i, root in enumerate(unscored):
        for k, sort in ((10, DOC_ASC), (1000, DOC_DESC), (100, [col_sort(img, "n", ffi.ORDER_DESC), DOC_ASC[0]])):
            run_both(gpu_ctx, img, P.make_plan(root, k, sort), ctx=f"unscored {i} k={k}")
    run_both(gpu_ctx, img, P.make_plan(pp(["alpha", "be"], ffi.OCCUR_MUST), 0, DOC_DESC, aggs=[terms_agg(img, "n")]),
             ctx="phrase prefix + terms agg")
    # a batch mixing plain phrases and phrase prefixes
    plans = [P.make_plan(P.phrase(img, "body", ["alpha", "beta"]), 100, DOC_ASC),
             P.make_plan(pp(["alpha", "be"], ffi.OCCUR_MUST), 100, DOC_ASC),
             P.make_plan(P.phrase(img, "body", ["beta", "alpha", "gamma"]), 100, DOC_ASC)]
    for got, plan in zip(gpu_ctx.split_search([img.split_id] * 3, plans), plans):
        assert_same(got, O.split_search(img, rewrite_as_phrases(plan)), ctx="mixed batch")


def test_synthetic_msg_field(gpu_ctx):
    img = S.synth_split(400_000, 7, [0.2, 0.05], split_id="synth-msg-pp", msg_vocab=64)
    gpu_ctx.register_split(img)
    try:
        assert len(P.prefix_expansions(img, "msg", "w1", 50)) == 11
        assert len(P.prefix_expansions(img, "msg", "w", 50)) == 50
        for tokens, m in ((["w0", "w1"], 50), (["w40", "w1"], 50), (["w1", "w2", "w3"], 50), (["w0", "w"], 50)):
            node = P.phrase_prefix(img, "msg", tokens, m)
            for k, sort in ((200, DOC_DESC), (10, [col_sort(img, "timestamp", ffi.ORDER_DESC)])):
                got = run_both(gpu_ctx, img, P.make_plan(node, k, sort), ctx=f"msg {tokens} k={k}")
            cross = gpu_ctx.split_search([img.split_id], [P.make_plan(or_plan(img, "msg", tokens, m), 10, [col_sort(img, "timestamp", ffi.ORDER_DESC)])])[0]
            assert (cross.num_hits, cross.hits) == (got.num_hits, got.hits), tokens
    finally:
        gpu_ctx.unregister_split(img.split_id)


def test_engine_refusals(gpu_ctx, pp_split):
    img = pp_split
    node = P.phrase_prefix(img, "body", ["alpha", "be"], 50)

    def code(plan):
        with pytest.raises(ffi.QwGpuError) as e:
            gpu_ctx.split_search([img.split_id], [plan])
        return e.value.code

    assert code(P.make_plan(node, 10, SCORE_DESC)) == ffi.EUNSUPPORTED  # a scored phrase prefix
    ords = P.prefix_expansions(img, "body", "a", 10)
    many = P.Node(ffi.NODE_PHRASE_PREFIX, children=[node.children[0]] + [P.Node(ffi.NODE_TERM, term_ord=ords[i % len(ords)], lo=1)
                                                                        for i in range(ffi.MAX_PREFIX_EXPANSIONS + 1)], lo=1)
    assert code(P.make_plan(many, 10, DOC_ASC)) == ffi.EUNSUPPORTED
    at_cap = P.Node(ffi.NODE_PHRASE_PREFIX, children=many.children[:-1], lo=1)
    run_both(gpu_ctx, img, P.make_plan(at_cap, 10, DOC_ASC), ctx="cap")
    kids = node.children

    def bad(children, lo):
        return P.make_plan(P.Node(ffi.NODE_PHRASE_PREFIX, children=children, lo=lo), 10, DOC_ASC)

    assert code(bad(kids, 0)) == ffi.EINVALID_ARG                       # no exact term
    assert code(bad(kids, len(kids))) == ffi.EINVALID_ARG               # no expansion
    assert code(bad(kids[:1], 1)) == ffi.EINVALID_ARG
    assert code(bad(kids, ffi.MAX_PHRASE_TERMS)) == ffi.EINVALID_ARG
    assert code(bad([kids[0], P.Node(ffi.NODE_TERM, lo=1)], 1)) == ffi.EINVALID_ARG  # absent term
    assert code(bad([kids[0], P.range_(img, "n", 0, 3)], 1)) == ffi.EINVALID_ARG
    tag = P.Node(ffi.NODE_TERM, term_ord=img.term_ord("tags", "beta"), lo=1)
    assert code(bad([kids[0], tag], 1)) == ffi.EINVALID_ARG             # terms of different fields
    shifted = P.Node(ffi.NODE_TERM, term_ord=kids[-1].term_ord, lo=2)
    assert code(bad(kids + [shifted], 1)) == ffi.EINVALID_ARG           # expansions at different offsets
    # a term offset beyond 32 bits, in a phrase prefix and in a plain phrase
    assert code(bad([kids[0], P.Node(ffi.NODE_TERM, term_ord=kids[-1].term_ord, lo=1 << 32)], 1)) == ffi.EINVALID_ARG
    far = P.Node(ffi.NODE_TERM, term_ord=kids[0].term_ord, lo=1 << 32)
    assert code(P.make_plan(P.Node(ffi.NODE_PHRASE, children=[kids[0], far]), 10, DOC_ASC)) == ffi.EINVALID_ARG


# ---- full request paths ------------------------------------------------------------------------------------

def gpu_root_search(ctx, imgs, query_ast, doc_mapper, **req_kw):
    leaf_pb = search_request(query_ast, **leafify(req_kw))
    root_pb = search_request(query_ast, **req_kw)
    offsets = [proto.enc_split_offsets(im.split_id, im.num_docs) for im in imgs]
    leaf_resp = ctx.leaf_search(proto.enc_leaf_search_request(leaf_pb, offsets, json.dumps(doc_mapper)))
    return proto.dec_leaf_search_response(service.merge_leaf_responses(root_pb, [leaf_resp]))


def test_gharchive_goldens_on_cuda(gpu_ctx):
    img = S.build_split(gharchive_docs(), GH_MAPPING, "gharchive")
    gpu_ctx.register_split(img)
    try:
        for field, phrase, m, want in GH_PHRASE_PREFIX_COUNTS:
            for kw in (dict(max_hits=0), dict(max_hits=20, sort_fields=[("_doc", DESC)])):
                got = gpu_root_search(gpu_ctx, [img], phrase_prefix_ast(field, phrase, m), GH_MAPPING, **kw)
                assert got["num_hits"] == want, (field, phrase, m)
        for text, op, want in GH_BOOL_PREFIX_COUNTS:
            got = gpu_root_search(gpu_ctx, [img], bool_prefix_ast(GH_BODY, text, op), GH_MAPPING, max_hits=5)
            assert got["num_hits"] == want, (text, op)
    finally:
        gpu_ctx.unregister_split(img.split_id)


def test_leaf_search_and_invoke_over_several_splits(gpu_ctx):
    imgs = [S.build_split(_docs(6000 + 500 * i, 100 + i), MAPPING, f"pp-leaf-{i}") for i in range(3)]
    for im in imgs:
        gpu_ctx.register_split(im)
    try:
        queries = [phrase_prefix_ast("body", "alpha be", 2), phrase_prefix_ast("body", "beta al"),
                   phrase_prefix_ast("body", "alt"), bool_prefix_ast("body", "gamma delta ga", "And", 3),
                   bool_(must=[term("body", "alpha")], filter=[phrase_prefix_ast("body", "beta ga")]),
                   {"type": "full_text", "field": "body", "text": "alpha beta",
                    "params": {"mode": {"type": "phrase", "slop": 0}}, "lenient": False}]
        for q in queries:
            for kw in (dict(max_hits=30, sort_fields=[("_doc", ASC)]), dict(max_hits=15, sort_fields=[("n", DESC)]),
                       dict(max_hits=0, aggs={"by_n": {"terms": {"field": "n", "size": 10}}})):
                got = gpu_root_search(gpu_ctx, imgs, q, MAPPING, **kw)
                want = cpu_root_search(imgs, q, MAPPING, **{k: v for k, v in kw.items() if k != "aggs"})
                assert got["num_hits"] == want["num_hits"] and got["partial_hits"] == want["partial_hits"], (q, kw)
        # search_after: the second page of a doc-id sorted phrase prefix
        q = phrase_prefix_ast("body", "alpha be")
        page1 = gpu_root_search(gpu_ctx, imgs, q, MAPPING, max_hits=40, sort_fields=[("_doc", ASC)])
        kw = dict(max_hits=40, sort_fields=[("_doc", ASC)], search_after=page1["partial_hits"][-1])
        page2 = gpu_root_search(gpu_ctx, imgs, q, MAPPING, **kw)
        assert page2["partial_hits"] == cpu_root_search(imgs, q, MAPPING, **kw)["partial_hits"]
        assert page2["partial_hits"] and page2["partial_hits"][0] != page1["partial_hits"][-1]
        # invoke_leaf_search: one batch, phrase prefixes and plain phrases side by side
        leaf_pb = search_request(bool_(should=[phrase_prefix_ast("body", "alpha be"), queries[-1]]), max_hits=25,
                                 sort_fields=[("_doc", DESC)])
        offsets = [proto.enc_split_offsets(im.split_id, im.num_docs) for im in imgs]
        results = proto.dec_lambda_responses(gpu_ctx.invoke_leaf_search(proto.enc_leaf_search_request(leaf_pb, offsets, json.dumps(MAPPING))))
        for im, r in zip(imgs, results):
            plan = rewrite_as_phrases(service.compile_plan(im, leaf_pb, json.dumps(MAPPING)))
            o = O.split_search(im, plan)
            want = proto.dec_leaf_search_response(service.build_leaf_response(im, leaf_pb, json.dumps(MAPPING), o.num_hits, o.hits, o.cells))
            assert r["response"]["num_hits"] == want["num_hits"] and r["response"]["partial_hits"] == want["partial_hits"]
        # under _score ranking a scoring phrase prefix is refused; in a filter it is served (above)
        bad = proto.enc_leaf_search_request(search_request(phrase_prefix_ast("body", "alpha be"), max_hits=5,
                                                           sort_fields=[("_score", DESC)]), offsets[:1], json.dumps(MAPPING))
        try:
            resp = proto.dec_leaf_search_response(gpu_ctx.leaf_search(bad))
            assert resp["num_successful_splits"] == 0 and len(resp["failed_splits"]) == 1
        except ffi.QwGpuError as e:
            assert e.code == ffi.EUNSUPPORTED
    finally:
        for im in imgs:
            gpu_ctx.unregister_split(im.split_id)
