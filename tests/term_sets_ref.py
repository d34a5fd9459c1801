"""Term sets, wildcards and one-token prefixes for the tests: the rewrite of a compiled plan's TERM_SET and COL_SET
nodes into bools of their children as should clauses (so that the CPU oracle, which has neither node, stands in for
the GPU engine), a splitgen corpus with a field of every kind a set can name, and a brute force over its documents.

Brute force (TermSetQuery, term_set_query.rs): a doc matches a `term_set` when one of its values on a named field
equals one of the field's literals, compared as the field indexes them: the raw text of a raw field, the tokens of a
default-tokenized field against the literal as given (a term_set never tokenizes it), the mapped-u64 value of a
numeric, bool or datetime column (datetime truncated to the field's fast_precision), the 16-byte form of an address."""
from __future__ import annotations

import ctypes as C
import json
from typing import Dict, List, Optional, Sequence

import numpy as np

from quickwit_b200 import ffi, plan as P, service, splitgen as S
from oracle import oracle as O
from pipeline import search_request
from regex_ref import parse_plan
import column_ref as R

SET_KINDS = (ffi.NODE_TERM_SET, ffi.NODE_COL_SET)


def rewrite_sets(plan: bytes) -> bytes:
    """The plan with every TERM_SET / COL_SET node replaced by a bool of its children as should clauses, and every
    CACHE node by its child (the oracle has none of the three)."""
    h, root, tail = parse_plan(plan)

    def rw(n):
        if n.kind in SET_KINDS:
            return P.Node(ffi.NODE_BOOL, n.occur, 1.0, children=n.children)
        if n.kind == ffi.NODE_CACHE:
            c = rw(n.children[0])
            c.occur = n.occur
            return c
        n.children = [rw(c) for c in n.children]
        return n

    nodes = P._flatten(rw(root))
    h.num_nodes = len(nodes)
    return bytes(h) + b"".join(bytes(n) for n in nodes) + tail


def oracle_search(img, plan: bytes):
    return O.split_search(img, rewrite_sets(plan))


def cpu_root_search(imgs: Sequence, query_ast, doc_mapper, **req_kw):
    """tests/pipeline.cpu_root_search with each split's compiled plan rewritten by rewrite_sets."""
    from quickwit_b200 import proto
    from pipeline import leafify
    dm = json.dumps(doc_mapper)
    leaf_pb = search_request(query_ast, **leafify(req_kw))
    root_pb = search_request(query_ast, **req_kw)
    parts = []
    for img in imgs:
        r = oracle_search(img, service.compile_plan(img, leaf_pb, dm))
        parts.append(service.build_leaf_response(img, leaf_pb, dm, r.num_hits, r.hits, r.cells))
    leaf_merged = service.merge_leaf_responses(leaf_pb, parts)
    return proto.dec_leaf_search_response(service.merge_leaf_responses(root_pb, [leaf_merged]))


def plan_nodes(plan: bytes) -> List[ffi.QwPlanNode]:
    hs, ns = C.sizeof(ffi.QwPlanHeader), C.sizeof(ffi.QwPlanNode)
    h = ffi.QwPlanHeader.from_buffer_copy(plan[:hs])
    return [ffi.QwPlanNode.from_buffer_copy(plan[hs + i * ns: hs + (i + 1) * ns]) for i in range(h.num_nodes)]


def node_bytes(plan: bytes) -> bytes:
    hs, ns = C.sizeof(ffi.QwPlanHeader), C.sizeof(ffi.QwPlanNode)
    h = ffi.QwPlanHeader.from_buffer_copy(plan[:hs])
    return plan[hs: hs + h.num_nodes * ns]


def set_nodes(plan: bytes) -> List[P.Node]:
    out, stack = [], [parse_plan(plan)[1]]
    while stack:
        n = stack.pop()
        if n.kind in SET_KINDS:
            out.append(n)
        else:
            stack.extend(n.children)
    return out


def compile_plan(img, ast, mapping, **kw) -> bytes:
    return service.compile_plan(img, search_request(ast, **kw), json.dumps(mapping))


def term_set(terms_per_field: Dict[str, Sequence]) -> dict:
    return {"type": "term_set", "terms_per_field": {k: list(v) for k, v in terms_per_field.items()}}


def wildcard(field: str, value: str) -> dict:
    return {"type": "wildcard", "field": field, "value": value}


def prefix(field: str, text: str, max_expansions: int) -> dict:
    return {"type": "phrase_prefix", "field": field, "phrase": text, "max_expansions": max_expansions}


def bool_prefix(field: str, text: str, max_expansions: int) -> dict:
    return {"type": "full_text", "field": field, "text": text,
            "params": {"mode": {"type": "bool_prefix", "max_expansions": max_expansions}}}


# ---- a corpus with every kind of set field -------------------------------------------------------------------------
MAPPING = {"field_mappings": [
    {"name": "raw", "type": "text", "tokenizer": "raw"},
    {"name": "body", "type": "text"},
    {"name": "u", "type": "u64", "fast": True},
    {"name": "i", "type": "i64", "fast": True},
    {"name": "f", "type": "f64", "fast": True},
    {"name": "b", "type": "bool", "fast": True},
    {"name": "dt", "type": "datetime", "fast": True, "fast_precision": "milliseconds"},
    {"name": "fo", "type": "text", "tokenizer": "raw", "fast": True, "indexed": False},
    {"name": "ipi", "type": "ip"},
    {"name": "ipf", "type": "ip", "fast": True, "indexed": False},
    {"name": "mu", "type": "u64", "fast": True},   # MULTI: 0..3 values per doc
    {"name": "ou", "type": "u64", "fast": True},   # OPTIONAL: ~half the docs
]}
N_DOCS = 3000
F64S = [float("-inf"), -1.5, -0.0, 0.0, 0.25, 1e300, float("inf")]
DT0 = 1_600_000_000_000  # ms since the epoch


def dt_text(ms: int) -> str:
    import datetime as _dt
    t = _dt.datetime.fromtimestamp(ms // 1000, tz=_dt.timezone.utc)
    return t.strftime("%Y-%m-%dT%H:%M:%S") + f".{ms % 1000:03d}Z"


def corpus_docs(seed: int = 7) -> List[dict]:
    rng = np.random.default_rng(seed)
    docs = []
    for d in range(N_DOCS):
        doc = {
            "raw": f"r{int(rng.integers(0, 400)):03d}",
            "body": f"Alpha w{int(rng.integers(0, 300))} beta",
            "u": int(rng.integers(0, 500)) * 7 + 11,
            "i": int(rng.integers(-300, 300)),
            "f": F64S[d % len(F64S)] if d % 3 else float(rng.integers(-50, 50)) / 4,
            "b": bool(rng.integers(0, 2)),
            "dt": dt_text(DT0 + int(rng.integers(0, 2000)) * 1000 + int(rng.integers(0, 3))),
            "fo": f"s{int(rng.integers(0, 300)):03d}",
            "ipi": f"10.0.{int(rng.integers(0, 2))}.{int(rng.integers(0, 256))}",
            "ipf": f"192.168.{int(rng.integers(0, 3))}.{int(rng.integers(0, 256))}",
            "mu": [int(x) for x in rng.integers(0, 600, size=int(rng.integers(0, 4)))],
        }
        if rng.random() < 0.5:
            doc["ou"] = int(rng.integers(0, 300))
        docs.append(doc)
    return docs


def _key(field: str, v):
    """A doc value or a literal as the field compares it; None: a literal that names no value."""
    if field in ("raw", "fo"):
        return str(v)
    if field in ("ipi", "ipf"):
        return S.parse_ip(str(v))
    if field in ("u", "mu", "ou"):
        return int(v)
    if field == "i":
        return S.i64_to_u64(int(v))
    if field == "f":
        return S.f64_to_u64(float(v))
    if field == "b":
        return (str(v).lower() == "true") if isinstance(v, str) else bool(v)
    if field == "dt":  # an integer literal here is in milliseconds (quickwit's timestamp autodetection)
        ns = int(v) * 1_000_000 if isinstance(v, int) else S.parse_datetime_nanos(v)
        return S.i64_to_u64(ns - ns % 1_000_000)
    raise KeyError(field)


def doc_keys(doc: dict, field: str) -> set:
    v = doc.get(field)
    vs = v if isinstance(v, list) else ([] if v is None else [v])
    if field == "body":
        return {t for x in vs for t in S.tokenize(str(x), "default")}
    return {_key(field, x) for x in vs}


def brute_term_set(docs: Sequence[dict], terms_per_field: Dict[str, Sequence]) -> np.ndarray:
    want = {f: ({str(x) for x in lits} if f == "body" else {_key(f, x) for x in lits}) for f, lits in terms_per_field.items()}
    return np.array([any(doc_keys(d, f) & w for f, w in want.items()) for d in docs], dtype=bool)


def hit_mask(res, n: int) -> np.ndarray:
    m = np.zeros(n, dtype=bool)
    m[[int(h[0]) for h in res.hits]] = True
    assert int(m.sum()) == res.num_hits
    return m


# ---- column_ref clauses with a set -----------------------------------------------------------------------------------
class SetQ(R.Q):
    """A set of mapped values on one column of a column_corpora split; as_bool: the same set as a bool of RANGE
    lo == hi should clauses."""

    def __init__(self, col: str, values: Sequence[int], occur: int = R.FILTER, as_bool: bool = False):
        super().__init__("set", occur, col=col)
        self.values, self.as_bool = [int(v) for v in values], as_bool

    def __repr__(self):
        return f"set[{self.occur}]({self.col}, {len(self.values)} values{', bool' if self.as_bool else ''})"


def node(sp, q) -> P.Node:
    if q.kind == "set":
        if q.as_bool:
            kids = [P.range_(sp.img, q.col, v, v, ffi.OCCUR_SHOULD) for v in sorted(set(q.values))]
            return P.bool_(kids, occur=q.occur)
        return P.col_set(sp.img, q.col, q.values, q.occur)
    if q.kind == "bool":
        return P.bool_([node(sp, c) for c in q.children], q.msm, q.occur)
    return R.node(sp, q)


def _leaf(sp, q):
    if q.kind != "set":
        return R._leaf(sp, q)
    c = sp.cols.get(q.col)
    m = np.zeros(sp.num_docs, dtype=bool)
    if c is not None:
        m[c.doc_of[np.isin(c.vals, np.array(q.values, dtype=np.uint64))]] = True
    return m, np.zeros(sp.num_docs, dtype=np.float32)


def evaluate(sp, q):
    import bool_ref
    return bool_ref.evaluate(q, lambda x: _leaf(sp, x), sp.num_docs)


def plan(sp, q, sort, K, sa=None, aggs=()) -> bytes:
    return P.make_plan(node(sp, q), K, sort.spec(sp), aggs=aggs, search_after=sa)


def probe_values(c, k: int, rs: np.random.Generator) -> List[int]:
    """k mapped values for a set on column c: stored values, one off them, between gcd multiples and outside
    [min, max], in about equal parts (fewer kinds for the smallest sets)."""
    U = (1 << 64) - 1
    stored = c.vals[rs.integers(0, c.vals.size, size=k)] if c.vals.size else np.zeros(k, dtype=np.uint64)
    out = []
    for j in range(k):
        s = int(stored[j])
        kind = j % 4
        if kind == 0:
            out.append(s)
        elif kind == 1:
            out.append(min(s + 1, U) if j % 8 == 1 else max(s - 1, 0))
        elif kind == 2:
            out.append(s + c.gcd // 2 if c.gcd > 1 and s + c.gcd // 2 <= U else s)
        else:
            out.append(U - j if c.max < U - j else (c.min - 1 - j if c.min > j else s))
    return out
