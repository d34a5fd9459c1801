"""Plain-Python restatement of quickwit's find_trace_ids collector (quickwit-search/src/find_trace_ids_collector.rs),
doc by doc: SelectTraceIds with its <= 2N map, truncation and sentinel, merge_segment_fruits, and the postcard bytes
of Vec<Span>. The tests compare the library against it; it shares no code with the library."""
from __future__ import annotations

import heapq
from typing import Iterable, List, Optional, Sequence, Tuple

I64_MIN = -(1 << 63)
Span = Tuple[bytes, int]  # (16-byte trace id, span timestamp in ns)


def span_key(s: Span):
    """Span::cmp: timestamp descending, then trace id bytes ascending."""
    return (-s[1], s[0])


class SelectTraceIds:
    def __init__(self, num_traces: int):
        self.n = num_traces
        self.map = {}
        self.workbench: List[Tuple[int, int]] = []
        self.running: Optional[int] = None
        self.running_ts = 0
        self.sentinel = I64_MIN

    def collect(self, ord_: int, ts: int):
        if self.running is None:
            self.running, self.running_ts = ord_, ts
            return
        if self.sentinel >= ts:
            return
        if self.running == ord_:
            self.running_ts = max(self.running_ts, ts)
        else:
            self._dedup(self.running, self.running_ts)
            self._truncate()
            self.running, self.running_ts = ord_, ts

    def _dedup(self, ord_, ts):
        if ord_ not in self.map or self.map[ord_] < ts:
            self.map[ord_] = ts

    def _select(self):
        if self.n == 0 or not self.map:
            return
        items = sorted(((o, t) for o, t in self.map.items()), key=lambda x: (-x[1], x[0]))
        self.map = {}
        k = min(self.n, len(items))
        self.workbench = items[:k]
        self.sentinel = self.workbench[k - 1][1]

    def _truncate(self):
        if len(self.map) < 2 * self.n:
            return
        self._select()
        for o, t in self.workbench[:self.n]:
            self.map[o] = t
        self.workbench = self.workbench[self.n:]

    def harvest(self) -> List[Tuple[int, int]]:
        if self.running is not None:
            self._dedup(self.running, self.running_ts)
            self.running = None
        self._select()
        return sorted(self.workbench, key=lambda x: (-x[1], x[0]))


def select_trace_ids(docs: Iterable[Tuple[int, int]], num_traces: int) -> List[Tuple[int, int]]:
    """(ordinal, timestamp) of the matched docs in doc order -> the split's [(ordinal, timestamp)], best first."""
    s = SelectTraceIds(num_traces)
    for o, t in docs:
        s.collect(o, t)
    return s.harvest()


def merge_segment_fruits(fruits: Sequence[Sequence[Span]], num_traces: int) -> List[Span]:
    out: List[Span] = []
    seen = set()
    if num_traces == 0:
        return out
    for sp in heapq.merge(*[sorted(f, key=span_key) for f in fruits], key=span_key):
        if sp[0] not in seen:
            seen.add(sp[0])
            out.append(sp)
            if len(out) == num_traces:
                break
    return out


def _varint(v: int) -> bytes:
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def encode_spans(spans: Sequence[Span]) -> bytes:
    """postcard of Vec<Span>: varint length, then 16 raw bytes + zigzag varint of the i64 per span."""
    out = bytearray(_varint(len(spans)))
    for tid, ts in spans:
        assert len(tid) == 16
        out += tid
        out += _varint(((ts << 1) ^ (ts >> 63)) & 0xFFFFFFFFFFFFFFFF)
    return bytes(out)


def split_spans(doc_ords_ts: Iterable[Tuple[int, int]], dictionary: Sequence[bytes], num_traces: int) -> List[Span]:
    """One split's fruit as the library emits it (sorted): trace ordinals mapped through the column dictionary."""
    return sorted(((dictionary[o], t) for o, t in select_trace_ids(doc_ords_ts, num_traces)), key=span_key)
