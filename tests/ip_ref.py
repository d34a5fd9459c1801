"""Brute force for `ip` fields, computed from the documents' address strings with Python's `ipaddress`.

Order and equality come from `ipaddress` (an IPv4 value is compared as its IPv4-mapped IPv6 form ::ffff:a.b.c.d, as
the reference's `into_ipv6_addr` stores it). The key rendering of a terms bucket is restated here rather than taken
from `str()`: an IPv4-mapped address renders as its dotted quad, any other as Rust's `Ipv6Addr` Display (RFC 5952),
while Python prints `::ffff:1.2.3.4` as `::ffff:102:304` on some versions.

Documents are dicts; a field's value is an address string or a list of them (multi-valued), absent when missing."""
from __future__ import annotations

import ipaddress
from typing import Dict, Iterable, List, Optional, Sequence, Tuple


def v6(text: str) -> ipaddress.IPv6Address:
    a = ipaddress.ip_address(text)
    return ipaddress.IPv6Address(b"\0" * 10 + b"\xff\xff" + a.packed) if a.version == 4 else a


def packed(text: str) -> bytes:
    return v6(text).packed


def render(a: ipaddress.IPv6Address) -> str:
    if a.ipv4_mapped is not None:
        return ".".join(str(b) for b in a.ipv4_mapped.packed)
    seg = [int.from_bytes(a.packed[2 * i:2 * i + 2], "big") for i in range(8)]
    best, best_len, cur, cur_len = 0, 0, 0, 0
    for i, s in enumerate(seg):
        if s == 0:
            if cur_len == 0:
                cur = i
            cur_len += 1
            if cur_len > best_len:  # the first longest run
                best, best_len = cur, cur_len
        else:
            cur_len = 0
    hexs = [format(s, "x") for s in seg]
    if best_len > 1:
        return ":".join(hexs[:best]) + "::" + ":".join(hexs[best + best_len:])
    return ":".join(hexs)


def values(doc: dict, field: str) -> List[ipaddress.IPv6Address]:
    v = doc.get(field)
    if v is None:
        return []
    return [v6(x) for x in (v if isinstance(v, list) else [v])]


def term_docs(docs: Sequence[dict], field: str, text: str) -> List[int]:
    a = v6(text)
    return [d for d, doc in enumerate(docs) if a in values(doc, field)]


def range_docs(docs: Sequence[dict], field: str, lo: Optional[str], hi: Optional[str], lo_incl: bool = True,
               hi_incl: bool = True) -> List[int]:
    """Docs holding at least one value inside the range; None = unbounded."""
    def inside(a):
        if lo is not None and (a < v6(lo) if lo_incl else a <= v6(lo)):
            return False
        if hi is not None and (a > v6(hi) if hi_incl else a >= v6(hi)):
            return False
        return True
    return [d for d, doc in enumerate(docs) if any(inside(a) for a in values(doc, field))]


def exists_docs(docs: Sequence[dict], field: str) -> List[int]:
    return [d for d, doc in enumerate(docs) if values(doc, field)]


def terms_counts(splits: Iterable[Tuple[Sequence[dict], Iterable[int]]], field: str,
                 missing: Optional[str] = None) -> Dict[ipaddress.IPv6Address, int]:
    """Bucket counts over the matched docs of every split: one count per value (a doc holding an address twice counts
    twice, as the column does), and the `missing` address for every matched doc without a value."""
    out: Dict[ipaddress.IPv6Address, int] = {}
    for docs, matched in splits:
        for d in matched:
            vs = values(docs[d], field)
            if not vs and missing is not None:
                vs = [v6(missing)]
            for a in vs:
                out[a] = out.get(a, 0) + 1
    return out


def terms_result(counts: Dict[ipaddress.IPv6Address, int], size: int = 10, order: str = "_count", desc: bool = True,
                 min_doc_count: int = 1) -> dict:
    """The finalised terms aggregation when no split cut a bucket (every split holds fewer distinct addresses than
    its segment size): buckets by count (ties by address ascending) or by address, the first `size` kept."""
    items = [(a, c) for a, c in counts.items() if c >= min_doc_count]
    if order == "_key":
        items.sort(key=lambda x: x[0], reverse=desc)
    else:
        items.sort(key=lambda x: (-x[1] if desc else x[1], x[0]))
    kept, rest = items[:size], items[size:]
    return {"buckets": [{"doc_count": c, "key": render(a)} for a, c in kept],
            "doc_count_error_upper_bound": 0, "sum_other_doc_count": sum(c for _, c in rest)}
