"""Composite aggregation pages (DESIGN.md §4.4, composite): device time and copied-back entry bytes of each page of
composite(terms(service), date_histogram(1h), terms(level)) with size 1000, over --splits splits of --docs log docs
(32 x 3.125 M by default, the size of the config-5 corpus), against the same tree as nested
terms(service) > date_histogram(1h) > terms(level) on the hashed path.

Corpus per split: a datetime column over one day at second precision, `service` (20 values, Zipf) and `level`
(5 values). Plans are built with plan.composite; each page's `after` is resolved per split into the node key spaces
the way the lowering does (terms: the raw value, histogram: the position relative to base_pos), from the last bucket
of the page before, which this script merges from the splits' entries.

Prints one JSON line per page and one for the nested tree: device time p50 / p99 of the call (CUDA events), the
entries copied back over all splits and their bytes (key record + cell per entry), the number of buckets of the page,
and the card name and power limit read in the same run. Nothing is written to the tree.

    python tools/bench_composite.py
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]

from quickwit_b200 import ffi, plan as P, splitgen as S  # noqa: E402
from quickwit_b200.service import SearcherContext  # noqa: E402

T0 = 1_700_000_000
HOUR_NS = 3600 * 10**9
ENTRY_BYTES = 48  # DHKey (16) + QwAggCell (32) per entry copied back


def build(split_ord, n, seed):
    rng = np.random.default_rng(seed + split_ord)
    ts = np.sort(rng.integers(0, 86_400, n)).astype(np.int64) * 10**9 + (T0 + 86_400 * split_ord) * 10**9
    b = S._Builder(n)
    b.add_column("timestamp", ffi.COL_DATETIME, ffi.CARD_FULL, ts.view(np.uint64) ^ np.uint64(1 << 63), None)
    b.add_column("service", ffi.COL_U64, ffi.CARD_FULL, np.minimum(rng.zipf(1.5, n) - 1, 19).astype(np.uint64), None)
    b.add_column("level", ffi.COL_U64, ffi.CARD_FULL, rng.integers(0, 5, n, dtype=np.uint64), None)
    return b.finish(f"composite-{split_ord:03d}")


class SplitAxes:
    """A split's three source nodes: their Agg, and the mapping between global keys and the node key spaces."""

    def __init__(self, img):
        self.img = img
        hdr = img.columns()
        self.cols = {c: img.column_ord(c) for c in ("timestamp", "service", "level")}
        self.h = {c: hdr[self.cols[c]] for c in self.cols}
        t = self.h["timestamp"]
        lo, hi = (S.u64_to_i64(v) for v in (t.min_value, t.max_value))
        self.base, self.nb = lo // HOUR_NS, hi // HOUR_NS - lo // HOUR_NS + 1

    def terms(self, name, *children):
        h = self.h[name]
        return P.Agg(ffi.AGG_TERMS, column=self.cols[name], num_buckets=(h.max_value - h.min_value) // h.gcd + 1, children=children)

    def hist(self, *children):
        return P.Agg(ffi.AGG_HISTOGRAM, column=self.cols["timestamp"], num_buckets=int(self.nb), interval=float(HOUR_NS),
                     base_pos=int(self.base), children=children)

    def terms_bound(self, name, v):  # ascending: smallest raw key not before v
        h = self.h[name]
        if v > h.max_value:
            return 0, ffi.AGG_COMP_AFTER_ALL
        if v < h.min_value:
            return 0, 0
        d = v - h.min_value
        return -(-d // h.gcd), ffi.AGG_COMP_EXACT if d % h.gcd == 0 else 0

    def hist_bound(self, pos):
        idx = pos - self.base
        if idx >= self.nb:
            return 0, ffi.AGG_COMP_AFTER_ALL
        return (0, 0) if idx < 0 else (int(idx), ffi.AGG_COMP_EXACT)

    def key(self, name, raw):
        h = self.h[name]
        return h.min_value + h.gcd * raw

    def composite_plan(self, size, after):
        srcs = [self.terms("service"), self.hist(), self.terms("level")]
        bounds = None
        if after is not None:
            bounds = [self.terms_bound("service", after[0]), self.hist_bound(after[1]), self.terms_bound("level", after[2])]
        return P.make_plan(P.bool_([P.match_all()]), 0, aggs=[P.composite(srcs, size, after=bounds)])

    def nested_plan(self):
        return P.make_plan(P.bool_([P.match_all()]), 0, aggs=[self.terms("service", self.hist(self.terms("level")))])

    def tuples(self, entries):
        """{(service, hour position, level): doc_count} of a composite result's leaves"""
        out = {}
        for node, parent, key, _f, cell in entries:
            if node != 2:
                continue
            hour = entries[parent]
            svc = entries[hour[1]]
            t = (self.key("service", svc[2]), self.base + hour[2], self.key("level", key))
            out[t] = out.get(t, 0) + cell[0]
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--splits", type=int, default=32)
    ap.add_argument("--docs", type=int, default=3_125_000)
    ap.add_argument("--size", type=int, default=1000)
    ap.add_argument("--pages", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    ctx = SearcherContext(0)
    t = time.time()
    axes = []
    for i in range(a.splits):
        img = build(i, a.docs, 0x5EED)
        ctx.register_split(img)
        axes.append(SplitAxes(img))
    build_s = time.time() - t
    ids = [x.img.split_id for x in axes]

    def timed(plans):
        times, res = [], None
        for step in range(a.warmup + a.steps):
            res = ctx.split_search(ids, plans)
            assert res[0].kernel_mask & ffi.KERNEL_HASHED_AGGS, hex(res[0].kernel_mask)
            if step >= a.warmup:
                times.append(res[0].gpu_time_us)
        return times, res

    def line(workload, times, res, **kw):
        n = sum(r.num_entries for r in res)
        print(json.dumps({"workload": workload, "splits": a.splits, "docs_per_split": a.docs,
                          "device_us_p50": float(np.percentile(times, 50)), "device_us_p99": float(np.percentile(times, 99)),
                          "calls": a.steps, "entries_copied_back": n, "d2h_entry_bytes": n * ENTRY_BYTES, **kw,
                          "gpu": gpu[0] if gpu else "unknown", "build_s": round(build_s, 1)}), flush=True)

    after = None
    for page in range(a.pages):
        times, res = timed([x.composite_plan(a.size, after) for x in axes])
        assert res[0].kernel_mask & ffi.KERNEL_COMPOSITE_CUT, hex(res[0].kernel_mask)
        merged = {}
        for x, r in zip(axes, res):
            for k, c in x.tuples(r.entries).items():
                merged[k] = merged.get(k, 0) + c
        keys = sorted(k for k in merged if after is None or k > after)[:a.size]
        line("composite_page", times, res, page=page, size=a.size, buckets=len(keys))
        if len(keys) < a.size:
            break
        after = keys[-1]
    times, res = timed([x.nested_plan() for x in axes])
    line("nested_terms_date_histogram_terms", times, res)
    ctx.close()


if __name__ == "__main__":
    main()
