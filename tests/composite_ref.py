"""The composite aggregation restated from documents: every key tuple the docs reach, in the sources' order, with
the docs of each bucket; then `after` and the cut to `size`. And, for host tests, the engine entries (QwAggEntry
tuples) of one split's source chain, built from the split image's column headers and dictionaries.

Keys: terms = the field's value (str / int / float / bool); histogram = floor((v - offset) / interval) * interval +
offset as a float; date_histogram over epoch seconds = the bucket's epoch milliseconds as an int; a doc without a value
gets None with `missing_bucket`, else no bucket. Ascending order puts None first, descending last."""
from __future__ import annotations

import functools
import itertools
import math
from typing import Any, Dict, List, Optional, Sequence, Tuple

from quickwit_b200 import ffi, splitgen as S


def sources_of(spec: Dict[str, Any]) -> List[Tuple[str, str, Dict[str, Any]]]:
    """[(name, type, params)] of a composite request body."""
    return [(name, t, p) for s in spec["sources"] for name, body in s.items() for t, p in body.items()]


def _vals(doc, field):
    v = doc.get(field)
    if v is None:
        return []
    return list(v) if isinstance(v, list) else [v]


def _dur_ms(s: str) -> int:
    units = {"ms": 1, "s": 1000, "m": 60000, "h": 3600000, "d": 86400000}
    for u in ("ms", "s", "m", "h", "d"):
        if s.endswith(u) and s[:-len(u)].lstrip("-").isdigit():
            return int(s[:-len(u)]) * units[u]
    raise ValueError(s)


def doc_keys(doc, t: str, p: Dict[str, Any]) -> List[Any]:
    vals = _vals(doc, p["field"])
    if t == "terms":
        keys = vals
    elif t == "histogram":
        iv, off = float(p["interval"]), float(p.get("offset", 0))
        keys = [math.floor((float(x) - off) / iv) * iv + off for x in vals]
    else:  # date_histogram over epoch seconds
        iv, off = _dur_ms(p["fixed_interval"]), _dur_ms(p["offset"]) if "offset" in p else 0
        keys = [((int(x) * 1000 - off) // iv) * iv + off for x in vals]
    if not keys:
        return [None] if p.get("missing_bucket") else []
    return keys


def _cmp1(a, b, desc: bool) -> int:
    if a is None or b is None:
        c = (a is not None) - (b is not None)
    else:
        c = (a > b) - (a < b)
    return -c if desc else c


def tuple_cmp(srcs, x, y) -> int:
    for (_n, _t, p), a, b in zip(srcs, x, y):
        c = _cmp1(a, b, p.get("order") == "desc")
        if c:
            return c
    return 0


def all_buckets(docs: Sequence[dict], spec: Dict[str, Any]) -> List[Tuple[tuple, List[dict]]]:
    """Every (key tuple, docs) in order; a doc appears once per value combination that reaches the tuple."""
    srcs = sources_of(spec)
    out: Dict[tuple, List[dict]] = {}
    for d in docs:
        for combo in itertools.product(*[doc_keys(d, t, p) for _n, t, p in srcs]):
            out.setdefault(combo, []).append(d)
    keys = sorted(out, key=functools.cmp_to_key(lambda x, y: tuple_cmp(srcs, x, y)))
    return [(k, out[k]) for k in keys]


def page(docs: Sequence[dict], spec: Dict[str, Any]) -> List[Tuple[tuple, List[dict]]]:
    """The buckets a composite request returns: those after `after`, cut to `size`."""
    srcs = sources_of(spec)
    bs = all_buckets(docs, spec)
    if "after" in spec:
        after = tuple(plain_after(spec["after"][n]) for n, _t, _p in srcs)
        bs = [b for b in bs if tuple_cmp(srcs, b[0], after) > 0]
    return bs[:spec.get("size", 10)]


def plain_after(v):
    """A type-tagged after_key value as the plain value it stands for."""
    if isinstance(v, str) and ":" in v:
        tag, rest = v.split(":", 1)
        if tag == "str":
            return rest
        if tag in ("i64", "u64"):
            return int(rest)
        if tag == "f64":
            return float(rest)
        if tag == "bool":
            return rest == "true"
    return v


def as_json(buckets, spec, sub=None) -> List[dict]:
    """Buckets as the finalised JSON lists them (without sub-aggregations unless `sub(docs)` gives them)."""
    names = [n for n, _t, _p in sources_of(spec)]
    out = []
    for k, ds in buckets:
        b = {"doc_count": len(ds), "key": dict(zip(names, k))}
        if sub:
            b.update(sub(ds))
        out.append(b)
    return out


# ---- engine entries of one split (host tests) ---------------------------------------------------------------------
def split_entries(img, plan: bytes, docs: Sequence[dict], spec: Dict[str, Any]) -> List[tuple]:
    """QwAggEntry tuples (node, parent, key, flags, cell) of a plan whose only aggregation is the composite (sources
    lowered to nodes 0..n-1), for every doc of the split, as the hashed walk emits them without an `after` filter."""
    h = ffi.QwPlanHeader.from_buffer_copy(plan)
    off = ffi.C.sizeof(ffi.QwPlanHeader) + h.num_nodes * ffi.C.sizeof(ffi.QwPlanNode)
    nodes = [ffi.QwAggNode.from_buffer_copy(plan, off + i * ffi.C.sizeof(ffi.QwAggNode)) for i in range(h.num_aggs)]
    hdr = img.columns()
    srcs = sources_of(spec)

    def raw_keys(i, d) -> List[Tuple[int, int]]:
        n, (_name, t, p) = nodes[i], srcs[i]
        vals = _vals(d, p["field"]) if n.column != ffi.ABSENT else []
        out = []
        if vals:
            c = hdr[n.column]
            for v in vals:
                if c.type == ffi.COL_STR:
                    m = img.dictionary(n.column).index(str(v).encode())
                elif c.type == ffi.COL_I64:
                    m = S.i64_to_u64(int(v))
                elif c.type == ffi.COL_F64:
                    m = S.f64_to_u64(float(v))
                else:
                    m = int(v)
                if t == "terms":
                    out.append(((m - c.min_value) // c.gcd, 0))
                else:
                    x = float(S.u64_to_i64(m)) if c.type == ffi.COL_I64 else (S.u64_to_f64(m) if c.type == ffi.COL_F64 else float(m))
                    out.append((math.floor((x - n.offset) / n.interval) - n.base_pos, 0))
        if not out and n.has_missing:
            out = [(0, ffi.AGG_ENTRY_MISSING)]
        return out

    # (a prefix entry carries the count of the leaves below it: the builder reads the leaves' counts only)
    full: Dict[tuple, int] = {}
    for d in docs:
        for combo in itertools.product(*[raw_keys(i, d) for i in range(len(srcs))]):
            for lvl in range(len(srcs)):
                full[combo[:lvl + 1]] = full.get(combo[:lvl + 1], 0) + 1
    entries: List[tuple] = []
    ids: Dict[tuple, int] = {}
    for path in sorted(full, key=len):
        parent = ffi.AGG_NO_PARENT if len(path) == 1 else ids[path[:-1]]
        key, flags = path[-1]
        ids[path] = len(entries)
        entries.append((len(path) - 1, parent, key, flags, (full[path], 0, (1 << 64) - 1, 0)))
    return entries
