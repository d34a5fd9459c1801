"""Regex queries on the GPU: QW_NODE_TERM_SET through the k_term_set pre-pass and the window program's OP_TERM_SET,
checked bit for bit against the CPU oracle (which evaluates the same plan with each term set rewritten as an OR of its
terms) or, for the widest sets, against a Python doc set; and the reference's REST goldens through the leaf search."""
import json

import pytest

from quickwit_b200 import ffi, plan as P, proto, service, splitgen as S
from quickwit_b200.proto import ASC, DESC
from helpers import DOC_ASC, DOC_DESC, SCORE_DESC, assert_same, col_sort, histogram_agg, terms_agg
from pipeline import bool_, leafify, search_request, term
from regex_ref import GH_MAPPING, GH_REGEX_COUNTS, cpu_root_search, dictionary, gharchive_docs, oracle_search, regex_ast

pytestmark = pytest.mark.gpu

@pytest.fixture(scope="module", autouse=True)
def _deep_limit(gpu_ctx):
    """K above 4096 (the deep selection path) needs the context's limit raised; restored afterwards."""
    gpu_ctx.set_max_hits(20_000)
    yield
    gpu_ctx.set_max_hits(4096)


# 100 003 docs: neither a multiple of 32 nor of any window size; `msg` holds w0 .. w63
N_SYNTH = 100_003


@pytest.fixture(scope="module")
def synth(gpu_ctx):
    img = S.synth_split(N_SYNTH, 3, [0.2, 0.05, 0.01], split_id="regex-synth", msg_vocab=64)
    gpu_ctx.register_split(img)
    yield img
    gpu_ctx.unregister_split(img.split_id)


def ts_(img, field, pattern, occur=ffi.OCCUR_FILTER):
    ords, _ = service.regex_terms(img, field, pattern)
    return P.term_set(img, field, ords, occur)


def run_both(ctx, img, plan, label):
    got = ctx.split_search([img.split_id], [plan])[0]
    assert_same(got, oracle_search(img, plan), ctx=label)
    return got


def test_term_set_as_every_clause(gpu_ctx, synth):
    img = synth
    t = lambda name, occ: P.term(img, "body", name, occur=occ)
    rng = lambda occ=ffi.OCCUR_FILTER: P.range_(img, "timestamp", 0, (1 << 64) - 1, occur=occ)
    day = img.column_ord("timestamp")
    assert day >= 0
    sparse, dense, mid = "w6[0-3]", "w.*", "w1.*"
    assert len(service.regex_terms(img, "msg", "w1.*")[0]) == 11 and len(service.regex_terms(img, "msg", dense)[0]) == 64
    roots = {
        "must": ts_(img, "msg", mid, ffi.OCCUR_MUST),
        "filter+term": P.bool_([t("t1", ffi.OCCUR_MUST), ts_(img, "msg", mid)]),
        "should": P.bool_([ts_(img, "msg", sparse, ffi.OCCUR_SHOULD), t("t2", ffi.OCCUR_SHOULD)]),
        "should msm": P.bool_([ts_(img, "msg", sparse, ffi.OCCUR_SHOULD), ts_(img, "msg", "w[0-2]", ffi.OCCUR_SHOULD),
                               t("t1", ffi.OCCUR_SHOULD)], min_should_match=2),
        "must_not": P.bool_([t("t0", ffi.OCCUR_MUST), ts_(img, "msg", mid, ffi.OCCUR_MUST_NOT)]),
        "two sets": P.bool_([ts_(img, "msg", "w[13].*"), ts_(img, "msg", "w[2-5]", ffi.OCCUR_MUST_NOT), rng()]),
        "dense": P.bool_([ts_(img, "msg", dense), t("t2", ffi.OCCUR_MUST)]),
        "nested": P.bool_([P.bool_([ts_(img, "msg", sparse, ffi.OCCUR_SHOULD), t("t0", ffi.OCCUR_SHOULD)], occur=ffi.OCCUR_MUST),
                           ts_(img, "msg", "w5.*", ffi.OCCUR_MUST_NOT)]),
    }
    n_hits = {}
    for name, root in roots.items():
        for k, sort in ((0, DOC_DESC), (10, DOC_ASC), (1000, DOC_DESC), (5000, DOC_ASC),
                        (20, [col_sort(img, "timestamp", ffi.ORDER_DESC)]), (50, [col_sort(img, "timestamp", ffi.ORDER_ASC), DOC_ASC[0]])):
            got = run_both(gpu_ctx, img, P.make_plan(root, k, sort), f"{name} k={k}")
            assert got.kernel_mask & ffi.KERNEL_TERM_SET and got.kernel_mask & ffi.KERNEL_WINDOW
            n_hits[name] = got.num_hits
        aggs = [terms_agg(img, "tenant_id") if img.column_ord("tenant_id") >= 0 else histogram_agg(img, "timestamp", 3600e9),
                histogram_agg(img, "timestamp", 3600e9)]
        run_both(gpu_ctx, img, P.make_plan(root, 0, DOC_DESC, aggs=aggs), f"{name} aggs")
        run_both(gpu_ctx, img, P.make_plan(root, 10, DOC_DESC, aggs=aggs[1:]), f"{name} hits + aggs")
    assert all(0 < n < N_SYNTH for n in n_hits.values()), n_hits


def test_term_set_beside_scored_terms(gpu_ctx, synth):
    img = synth
    t = lambda name, occ: P.term(img, "body", name, occur=occ)
    roots = [P.bool_([t("t0", ffi.OCCUR_SHOULD), t("t2", ffi.OCCUR_SHOULD), ts_(img, "msg", "w1.*")]),
             P.bool_([t("t1", ffi.OCCUR_MUST), ts_(img, "msg", "w[0-4]", ffi.OCCUR_MUST_NOT)]),
             P.bool_([t("t0", ffi.OCCUR_MUST), ts_(img, "msg", "w.*"), P.range_(img, "timestamp", 0, (1 << 64) - 1)])]
    for i, root in enumerate(roots):
        for k in (10, 1000, 6000):
            run_both(gpu_ctx, img, P.make_plan(root, k, SCORE_DESC), f"scored {i} k={k}")
    # search_after on a doc-id sort: the page after the 100th hit
    root = ts_(img, "msg", "w1.*", ffi.OCCUR_MUST)
    first = gpu_ctx.split_search([img.split_id], [P.make_plan(root, 100, DOC_ASC)])[0]
    sa = ffi.QwSearchAfter()
    sa.present, sa.has_v1, sa.v1 = 1, 1, first.hits[-1][0]
    run_both(gpu_ctx, img, P.make_plan(root, 100, DOC_ASC, search_after=sa), "search_after")


def test_engine_refusals(gpu_ctx, synth):
    img = synth
    node = ts_(img, "msg", "w1.*", ffi.OCCUR_MUST)

    def code(plan):
        with pytest.raises(ffi.QwGpuError) as e:
            gpu_ctx.split_search([img.split_id], [plan])
        return e.value.code

    assert code(P.make_plan(node, 10, SCORE_DESC)) == ffi.EUNSUPPORTED  # a scored term set
    kids = node.children
    bad = lambda children: P.make_plan(P.Node(ffi.NODE_TERM_SET, children=children), 10, DOC_ASC)
    assert code(bad([])) == ffi.EINVALID_ARG
    assert code(bad(kids[::-1])) == ffi.EINVALID_ARG                         # not increasing
    assert code(bad([kids[0], kids[0]])) == ffi.EINVALID_ARG                 # repeated
    assert code(bad([kids[0], P.Node(ffi.NODE_TERM)])) == ffi.EINVALID_ARG   # absent term
    assert code(bad([kids[0], P.range_(img, "timestamp", 0, 5)])) == ffi.EINVALID_ARG
    other = P.term(img, "body", "t0", occur=ffi.OCCUR_SHOULD)
    assert code(bad([other] + kids if other.term_ord < kids[0].term_ord else kids + [other])) == ffi.EINVALID_ARG


# ---- expansion sizes 1, 64, 4096, 65 536 over a wide field -----------------------------------------------------------
WIDE_MAPPING = {"field_mappings": [{"name": "tok", "type": "text"}, {"name": "n", "type": "u64", "fast": True}]}
N_WIDE = 22_001


@pytest.fixture(scope="module")
def wide(gpu_ctx):
    docs = [{"tok": " ".join(f"a{(3 * i + j) % 65536:05d}" for j in range(3)) + (" rare" if i % 997 == 5 else ""), "n": i % 37}
            for i in range(N_WIDE)]
    img = S.build_split(docs, WIDE_MAPPING, "regex-wide")
    gpu_ctx.register_split(img)
    yield img, [set(d["tok"].split()) for d in docs]
    gpu_ctx.unregister_split(img.split_id)


SIZES = [("a00000", 1), ("a000([0-5][0-9]|6[0-3])", 64), ("a(0[0-3][0-9]{3}|040[0-8][0-9]|0409[0-5])", 4096), ("a.*", 65536)]


@pytest.mark.parametrize("pattern,size", SIZES)
def test_expansion_sizes(gpu_ctx, wide, pattern, size):
    img, doc_tokens = wide
    ords, _ = service.regex_terms(img, "tok", pattern)
    assert len(ords) == size
    chosen = set(ords)
    words = {b.decode() for t, b in dictionary(img, "tok") if t in chosen}
    want = [d for d, toks in enumerate(doc_tokens) if toks & words]
    node = P.term_set(img, "tok", ords, ffi.OCCUR_MUST)
    for k, sort in ((0, DOC_DESC), (100, DOC_ASC), (4096, DOC_DESC), (8000, DOC_ASC)):
        got = gpu_ctx.split_search([img.split_id], [P.make_plan(node, k, sort)])[0]
        assert got.num_hits == len(want), (pattern, k)
        exp = want[:k] if sort is DOC_ASC else want[::-1][:k]
        assert [h[0] for h in got.hits] == exp, (pattern, k)
    if size <= 64:
        run_both(gpu_ctx, img, P.make_plan(node, 50, [col_sort(img, "n", ffi.ORDER_ASC)], aggs=[terms_agg(img, "n")]), pattern)
    # the dense case covers every document; a rare filter beside it
    if size == 65536:
        assert len(want) == N_WIDE
        root = P.bool_([P.term_set(img, "tok", ords, ffi.OCCUR_FILTER), P.term(img, "tok", "rare")])
        got = gpu_ctx.split_search([img.split_id], [P.make_plan(root, 100, DOC_ASC)])[0]
        assert [h[0] for h in got.hits] == [d for d in range(N_WIDE) if d % 997 == 5]


def test_batch_mask_and_launches(gpu_ctx, synth):
    """A batch without a term set runs as before; one with a term set adds exactly the pre-pass launch."""
    img = synth
    agg = [histogram_agg(img, "timestamp", 3600e9)]
    plain = P.make_plan(P.bool_([P.term(img, "body", "t1"), P.range_(img, "timestamp", 0, (1 << 64) - 1)]), 0, DOC_ASC, aggs=agg)
    other = P.make_plan(P.bool_([P.term(img, "body", "t0"), P.range_(img, "timestamp", 0, (1 << 64) - 1)]), 0, DOC_ASC, aggs=agg)
    with_set = P.make_plan(P.bool_([P.term(img, "body", "t0"), ts_(img, "msg", "w1.*")]), 0, DOC_ASC, aggs=agg)
    empty_set = P.make_plan(P.bool_([P.term(img, "body", "t0"), ts_(img, "msg", "zzz.*")]), 10, DOC_ASC, aggs=agg)
    a = gpu_ctx.split_search([img.split_id] * 2, [plain, other])
    b = gpu_ctx.split_search([img.split_id] * 2, [plain, with_set])
    assert not a[0].kernel_mask & ffi.KERNEL_TERM_SET
    assert b[0].kernel_mask == a[0].kernel_mask | ffi.KERNEL_TERM_SET
    assert b[0].num_kernel_launches == a[0].num_kernel_launches + 1
    for got, plan in zip(b, [plain, with_set]):
        assert_same(got, oracle_search(img, plan), ctx="mixed batch")
    # a split whose regex expands to nothing compiles to NONE: no pre-pass
    c = gpu_ctx.split_search([img.split_id], [empty_set])[0]
    assert not c.kernel_mask & ffi.KERNEL_TERM_SET and c.num_hits == 0


# ---- full request path ---------------------------------------------------------------------------------------------

def gpu_root_search(ctx, imgs, query_ast, doc_mapper, **req_kw):
    leaf_pb = search_request(query_ast, **leafify(req_kw))
    root_pb = search_request(query_ast, **req_kw)
    offsets = [proto.enc_split_offsets(im.split_id, im.num_docs) for im in imgs]
    leaf_resp = ctx.leaf_search(proto.enc_leaf_search_request(leaf_pb, offsets, json.dumps(doc_mapper)))
    return proto.dec_leaf_search_response(service.merge_leaf_responses(root_pb, [leaf_resp]))


def test_gharchive_goldens_on_cuda(gpu_ctx):
    img = S.build_split(gharchive_docs(), GH_MAPPING, "gharchive-regex")
    gpu_ctx.register_split(img)
    try:
        for field, regex, want in GH_REGEX_COUNTS:
            for kw in (dict(max_hits=0), dict(max_hits=20, sort_fields=[("_doc", DESC)])):
                got = gpu_root_search(gpu_ctx, [img], regex_ast(field, regex), GH_MAPPING, **kw)
                assert got["num_hits"] == want, (field, regex)
        # a regex filter under _score ranking is served; in a scoring clause the split fails
        q = bool_(must=[term("type", "pushevent")], filter=[regex_ast("repo.name", ".*[Rr]ust.*")])
        got = gpu_root_search(gpu_ctx, [img], q, GH_MAPPING, max_hits=5, sort_fields=[("_score", DESC)])
        want = cpu_root_search([img], q, GH_MAPPING, max_hits=5, sort_fields=[("_score", DESC)])
        assert got["num_hits"] == want["num_hits"] and got["partial_hits"] == want["partial_hits"]
        try:
            resp = gpu_root_search(gpu_ctx, [img], regex_ast("type", "push.*"), GH_MAPPING, max_hits=5, sort_fields=[("_score", DESC)])
            assert resp["num_successful_splits"] == 0 and len(resp["failed_splits"]) == 1
        except ffi.QwGpuError as e:
            assert e.code == ffi.EUNSUPPORTED
    finally:
        gpu_ctx.unregister_split(img.split_id)
