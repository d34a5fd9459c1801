"""Phrase-prefix restatements for the tests: a plain-Python scan of token lists, and the rewrite of a compiled plan's
PHRASE_PREFIX nodes into ORs of plain phrases (one per expansion) so that the CPU oracle, which evaluates plain
phrases, can stand in for the GPU engine."""
from __future__ import annotations

import ctypes as C
import gzip
import json
import os
from typing import Dict, List, Sequence, Tuple

from quickwit_b200 import ffi, plan as P, service
from oracle import oracle as O
from pipeline import leafify, search_request
from quickwit_b200 import proto

# a byte-for-byte copy of the reference's rest-api-tests/scenarii/es_compatibility/gharchive-bulk.json.gz
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gharchive-bulk.json.gz")
GH_BODY, GH_MSG = "payload.pull_request.body", "payload.commits.message"
GH_MAPPING = {"field_mappings": [{"name": GH_BODY, "type": "text", "record": "position"},
                                 {"name": GH_MSG, "type": "text", "record": "position"}]}
# rest-api-tests/scenarii/es_compatibility/0010-match_phrase_prefix_query.yaml, 0017-match-bool-prefix-query.yaml
GH_PHRASE_PREFIX_COUNTS = [(GH_BODY, "p", 50, 2), (GH_BODY, "to p", 50, 1), (GH_BODY, "be to p", 50, 1),
                           (GH_MSG, "automated comm", 50, 1), (GH_MSG, "fix", 2, 6), (GH_MSG, "fix", 50, 7)]
GH_BOOL_PREFIX_COUNTS = [("file not ch", "Or", 1), ("file not chzn", "And", 0), ("file not ch", "And", 1)]


def gharchive_docs() -> List[Dict]:
    """The two text paths of the reference's gharchive fixture, flattened (commit messages multi-valued)."""
    out = []
    with gzip.open(GOLDEN, "rt") as f:
        for line in f:
            d = json.loads(line)
            if "index" in d:
                continue
            p = d.get("payload", {})
            doc = {}
            body = (p.get("pull_request") or {}).get("body")
            if isinstance(body, str):
                doc[GH_BODY] = body
            msgs = [c["message"] for c in p.get("commits", []) or [] if isinstance(c.get("message"), str)]
            if msgs:
                doc[GH_MSG] = msgs
            out.append(doc)
    return out


def phrase_prefix_ast(field: str, phrase: str, max_expansions: int = 50, tokenizer=None, zero_terms_query="none",
                      lenient=False):
    params = {"mode": {"type": "phrase_fallback_to_intersection"}, "zero_terms_query": zero_terms_query}
    if tokenizer is not None:
        params["tokenizer"] = tokenizer
    return {"type": "phrase_prefix", "field": field, "phrase": phrase, "max_expansions": max_expansions,
            "params": params, "lenient": lenient}


def bool_prefix_ast(field: str, text: str, operator: str = "Or", max_expansions: int = 50, tokenizer=None):
    params = {"mode": {"type": "bool_prefix", "operator": operator, "max_expansions": max_expansions},
              "zero_terms_query": "none"}
    if tokenizer is not None:
        params["tokenizer"] = tokenizer
    return {"type": "full_text", "field": field, "text": text, "params": params, "lenient": False}


# ---- plan rewrite ------------------------------------------------------------------------------------

def parse_plan(plan: bytes) -> Tuple[ffi.QwPlanHeader, P.Node, bytes]:
    hs, ns = C.sizeof(ffi.QwPlanHeader), C.sizeof(ffi.QwPlanNode)
    h = ffi.QwPlanHeader.from_buffer_copy(plan[:hs])
    flat = [ffi.QwPlanNode.from_buffer_copy(plan[hs + i * ns: hs + (i + 1) * ns]) for i in range(h.num_nodes)]

    def node(i):
        n = flat[i]
        kids = [node(c) for c in range(n.first_child, n.first_child + n.num_children)] \
            if n.kind in (ffi.NODE_BOOL, ffi.NODE_PHRASE, ffi.NODE_PHRASE_PREFIX) else []
        return P.Node(n.kind, n.occur, n.boost, kids, None if n.min_should_match == ffi.ABSENT else n.min_should_match,
                      n.term_ord, n.field_id, n.bm25_weight, n.column, n.lo, n.hi)

    return h, node(0), plan[hs + h.num_nodes * ns:]


def phrase_prefix_nodes(root: P.Node) -> List[P.Node]:
    out, stack = [], [root]
    while stack:
        n = stack.pop()
        if n.kind == ffi.NODE_PHRASE_PREFIX:
            out.append(n)
        else:
            stack.extend(n.children)
    return out


def rewrite_as_phrases(plan: bytes) -> bytes:
    """The plan with every PHRASE_PREFIX node replaced by the OR of its plain phrases."""
    h, root, tail = parse_plan(plan)

    def rw(n):
        if n.kind == ffi.NODE_PHRASE_PREFIX:
            return P.phrase_prefix_as_phrases(n)
        n.children = [rw(c) for c in n.children] if n.kind == ffi.NODE_BOOL else n.children
        return n

    nodes = P._flatten(rw(root))
    h.num_nodes = len(nodes)
    return bytes(h) + b"".join(bytes(n) for n in nodes) + tail


def term_text(img, ord_: int) -> bytes:
    _h, _s, tbytes, _f, terms, _c = img._directory()
    t = terms[ord_]
    return bytes(tbytes[t.bytes_off: t.bytes_off + t.bytes_len])


def compiled_expansions(img, plan: bytes) -> List[bytes]:
    """The expansion terms a compiled plan carries: the last slot of its PHRASE_PREFIX node, or the TERM children
    of a one-token prefix's set filter."""
    _h, root, _t = parse_plan(plan)
    pp = phrase_prefix_nodes(root)
    if pp:
        assert len(pp) == 1
        return [term_text(img, c.term_ord) for c in pp[0].children[pp[0].lo:]]
    out, stack = [], [root]
    while stack:
        n = stack.pop()
        if n.kind == ffi.NODE_TERM and n.term_ord != ffi.ABSENT:
            out.append(n.term_ord)
        stack.extend(n.children)
    return [term_text(img, o) for o in sorted(out)]


def cpu_root_search(imgs: Sequence, query_ast, doc_mapper, **req_kw):
    """tests/pipeline.cpu_root_search with each split's compiled plan rewritten by rewrite_as_phrases."""
    dm = json.dumps(doc_mapper)
    leaf_pb = search_request(query_ast, **leafify(req_kw))
    root_pb = search_request(query_ast, **req_kw)
    parts = []
    for img in imgs:
        plan = rewrite_as_phrases(service.compile_plan(img, leaf_pb, dm))
        r = O.split_search(img, plan)
        parts.append(service.build_leaf_response(img, leaf_pb, dm, r.num_hits, r.hits, r.cells))
    leaf_merged = service.merge_leaf_responses(leaf_pb, parts)
    return proto.dec_leaf_search_response(service.merge_leaf_responses(root_pb, [leaf_merged]))


# ---- brute force -------------------------------------------------------------------------------------

def doc_positions(values: Sequence[str]) -> Dict[str, List[int]]:
    """token -> positions of one doc's values (default tokenizer, values one position apart)."""
    from quickwit_b200.splitgen import tokenize_default
    pos: Dict[str, List[int]] = {}
    start = 0
    for v in values:
        toks = tokenize_default(v)
        for i, t in enumerate(toks):
            pos.setdefault(t, []).append(start + i)
        start += len(toks) + 1
    return pos


def expansions(vocab: Sequence[str], prefix: str, max_expansions: int) -> List[str]:
    return [t for t in sorted(vocab, key=str.encode) if t.encode().startswith(prefix.encode())][:max_expansions]


def scan(doc_pos: Sequence[Dict[str, List[int]]], tokens: Sequence[str], exps: Sequence[str]) -> List[int]:
    """Doc ids that hold the phrase prefix: exact tokens at b + i, some expansion at b + k."""
    k = len(tokens) - 1
    out = []
    for d, pos in enumerate(doc_pos):
        if k == 0:
            hit = any(e in pos for e in exps)
        else:
            hit = any(all(b + i in pos.get(t, ()) for i, t in enumerate(tokens[:-1]))
                      for e in exps for q in pos.get(e, ()) for b in [q - k] if b >= 0)
        if hit:
            out.append(d)
    return out
