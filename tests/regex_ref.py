"""Regex restatements for the tests: a brute force (`re.fullmatch` over a split's decoded dictionary, for the served
subset), the gharchive fields the reference's regex scenarios query, and the rewrite of a compiled plan's TERM_SET
nodes into ORs of their TERM children, so that the CPU oracle (which has no term-set node) can stand in for the GPU
engine. The rewrite keeps the match set; the term set is never scored, and the tests only place it where its score is
not read."""
from __future__ import annotations

import ctypes as C
import gzip
import json
import re
from typing import Dict, List, Sequence, Tuple

from quickwit_b200 import ffi, plan as P, proto, service
from oracle import oracle as O
from phrase_prefix_ref import GOLDEN, term_text
from pipeline import leafify, search_request

GH_MAPPING = {"field_mappings": [{"name": "type", "type": "text"},
                                 {"name": "repo.name", "type": "text", "tokenizer": "raw"},
                                 {"name": "payload.description", "type": "text"}]}
# rest-api-tests/scenarii/es_compatibility/0031-regex.yaml and 0005-query_string_query.yaml (field, regex, hits);
# `case_insensitive: true` reaches the leaf as a leading (?i)
GH_REGEX_COUNTS = [("type", ".*event", 100), ("type", "event", 0), ("type", "pushevent", 60),
                   ("repo.name", "(?i)RUST.*", 1), ("repo.name", "RUST.*", 0), ("payload.description", "jour.*", 3)]


def gharchive_docs() -> List[Dict]:
    """`type`, `repo.name` and `payload.description` of the reference's gharchive fixture."""
    out = []
    with gzip.open(GOLDEN, "rt") as f:
        for line in f:
            d = json.loads(line)
            if "index" in d:
                continue
            doc = {"type": d.get("type")}
            name = (d.get("repo") or {}).get("name")
            if isinstance(name, str):
                doc["repo.name"] = name
            desc = (d.get("payload") or {}).get("description")
            if isinstance(desc, str):
                doc["payload.description"] = desc
            out.append({k: v for k, v in doc.items() if isinstance(v, str)})
    return out


def regex_ast(field: str, regex: str):
    return {"type": "regex", "field": field, "regex": regex}


# ---- plans -------------------------------------------------------------------------------------------

def parse_plan(plan: bytes) -> Tuple[ffi.QwPlanHeader, P.Node, bytes]:
    hs, ns = C.sizeof(ffi.QwPlanHeader), C.sizeof(ffi.QwPlanNode)
    h = ffi.QwPlanHeader.from_buffer_copy(plan[:hs])
    flat = [ffi.QwPlanNode.from_buffer_copy(plan[hs + i * ns: hs + (i + 1) * ns]) for i in range(h.num_nodes)]

    def node(i):
        n = flat[i]
        kids = [node(c) for c in range(n.first_child, n.first_child + n.num_children)] if n.kind != ffi.NODE_TERM else []
        return P.Node(n.kind, n.occur, n.boost, kids, None if n.min_should_match == ffi.ABSENT else n.min_should_match,
                      n.term_ord, n.field_id, n.bm25_weight, n.column, n.lo, n.hi)

    return h, node(0), plan[hs + h.num_nodes * ns:]


def term_set_nodes(root: P.Node) -> List[P.Node]:
    out, stack = [], [root]
    while stack:
        n = stack.pop()
        if n.kind == ffi.NODE_TERM_SET:
            out.append(n)
        else:
            stack.extend(n.children)
    return out


def compiled_expansions(img, plan: bytes) -> List[bytes]:
    """The terms of the compiled plan's one TERM_SET node (none when the regex compiled to match nothing)."""
    sets = term_set_nodes(parse_plan(plan)[1])
    assert len(sets) <= 1
    return [term_text(img, c.term_ord) for c in sets[0].children] if sets else []


def rewrite_term_sets(plan: bytes) -> bytes:
    """The plan with every TERM_SET node replaced by a bool of its TERM children as should clauses."""
    h, root, tail = parse_plan(plan)

    def rw(n):
        if n.kind == ffi.NODE_TERM_SET:
            return P.Node(ffi.NODE_BOOL, n.occur, 1.0, children=n.children)
        n.children = [rw(c) for c in n.children]
        return n

    nodes = P._flatten(rw(root))
    h.num_nodes = len(nodes)
    return bytes(h) + b"".join(bytes(n) for n in nodes) + tail


def oracle_search(img, plan: bytes):
    return O.split_search(img, rewrite_term_sets(plan))


def cpu_root_search(imgs: Sequence, query_ast, doc_mapper, **req_kw):
    """tests/pipeline.cpu_root_search with each split's compiled plan rewritten by rewrite_term_sets."""
    dm = json.dumps(doc_mapper)
    leaf_pb = search_request(query_ast, **leafify(req_kw))
    root_pb = search_request(query_ast, **req_kw)
    parts = []
    for img in imgs:
        r = oracle_search(img, service.compile_plan(img, leaf_pb, dm))
        parts.append(service.build_leaf_response(img, leaf_pb, dm, r.num_hits, r.hits, r.cells))
    leaf_merged = service.merge_leaf_responses(leaf_pb, parts)
    return proto.dec_leaf_search_response(service.merge_leaf_responses(root_pb, [leaf_merged]))


# ---- brute force -------------------------------------------------------------------------------------

def dictionary(img, field: str) -> List[Tuple[int, bytes]]:
    """(term ord, bytes) of one field, in dictionary order."""
    names = img.field_names()
    if field not in names:
        return []
    _h, _s, tbytes, fields, terms, _c = img._directory()
    f = fields[names.index(field)]
    return [(t, bytes(tbytes[terms[t].bytes_off: terms[t].bytes_off + terms[t].bytes_len]))
            for t in range(f.first_term, f.first_term + f.num_terms)]


def brute_force(img, field: str, py_pattern: str) -> List[bytes]:
    """Terms of `field` that Python's `re` matches whole. `py_pattern` must stay inside the served subset written
    the way Python reads it (Perl classes spelled as their ASCII classes, no U+0130 / U+0131 in the dictionary: Python
    folds `i` onto them under IGNORECASE, the reference's simple case folding does not)."""
    rx = re.compile(py_pattern)
    return [b for _t, b in dictionary(img, field) if rx.fullmatch(b.decode("utf-8"))]
