"""Aggregations in the hashed cell layout (DESIGN.md §4.4): device time of three dashboard queries that the dense
layout cannot serve, over --splits splits of --docs log docs (32 x 3.125 M by default, the size of the config-5 corpus).

Corpus per split: a datetime column over one day at second precision, `service` (20 values, Zipf), `level` (5 values),
`latency` (u64 < 2^20), `user_id` (u64 over the whole [0, 2^63] range, 50 000 distinct values) and `user_id_400k` (the
same range, 400 000 distinct values).
Queries (match_all, no hits, one call over every split):
  * nested: date_histogram(1h) > terms(service) > terms(level) > avg(latency)  — four levels;
  * wide:   terms(user_id) — a terms space far beyond 2^24 slots;
  * wide_retry: terms over a second user id column with 400 000 distinct values (almost all of them in every split), more than the
    initial capacity of 65536 cells: every call overflows, finishes its first pass early and runs again at the bound.

Prints one JSON line per query: device time p50 / p99 of the call (CUDA events), whether the capacity re-run ran, the
number of entries of split 0, and the card name and power limit read in the same run. Nothing is written to the tree.

    python tools/bench_nested_aggs.py
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


def build(split_ord, n, seed):
    rng = np.random.default_rng(seed + split_ord)
    ts = np.sort(rng.integers(0, 86_400, n)).astype(np.int64) * 10**9 + (T0 + 86_400 * split_ord) * 10**9
    users = rng.integers(0, 1 << 63, 50_000, dtype=np.uint64)
    users[:2] = [0, 1 << 63]
    b = S._Builder(n)
    b.add_column("timestamp", ffi.COL_DATETIME, ffi.CARD_FULL, ts.view(np.uint64) ^ np.uint64(1 << 63), None)
    b.add_column("service", ffi.COL_U64, ffi.CARD_FULL, np.minimum(rng.zipf(1.5, n) - 1, 19).astype(np.uint64), None)
    b.add_column("level", ffi.COL_U64, ffi.CARD_FULL, rng.integers(0, 5, n, dtype=np.uint64), None)
    b.add_column("latency", ffi.COL_U64, ffi.CARD_FULL, rng.integers(0, 1 << 20, n, dtype=np.uint64), None)
    b.add_column("user_id", ffi.COL_U64, ffi.CARD_FULL, rng.choice(users, n), None)
    many = rng.integers(0, 1 << 63, 400_000, dtype=np.uint64)
    many[:2] = [0, 1 << 63]
    b.add_column("user_id_400k", ffi.COL_U64, ffi.CARD_FULL, rng.choice(many, n), None)
    return b.finish(f"nested-{split_ord:03d}")


def plans_for(img, query):
    cols = {c: img.column_ord(c) for c in ("timestamp", "service", "level", "latency", "user_id", "user_id_400k")}
    hdr = img.columns()

    def terms(name, *children):
        h = hdr[cols[name]]
        nb = (h.max_value - h.min_value) // h.gcd + 1
        return P.Agg(ffi.AGG_TERMS, column=cols[name], num_buckets=min(nb, 0xFFFFFFFF), children=children)

    if query == "nested":
        h = hdr[cols["timestamp"]]
        lo, hi = (S.u64_to_i64(v) for v in (h.min_value, h.max_value))
        base, top = lo // HOUR_NS, hi // HOUR_NS
        aggs = [P.Agg(ffi.AGG_HISTOGRAM, column=cols["timestamp"], num_buckets=int(top - base + 1), interval=float(HOUR_NS),
                      base_pos=int(base), children=[terms("service", terms("level", P.Agg(ffi.AGG_STATS, column=cols["latency"])))])]
    elif query == "wide":
        aggs = [terms("user_id")]
    else:
        aggs = [terms("user_id_400k")]
    return P.make_plan(P.bool_([P.match_all()]), 0, aggs=aggs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--splits", type=int, default=32)
    ap.add_argument("--docs", type=int, default=3_125_000)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    ctx = SearcherContext(0)
    t = time.time()
    imgs = []
    for i in range(a.splits):
        img = build(i, a.docs, 0x5EED)
        ctx.register_split(img)
        imgs.append(img)
    build_s = time.time() - t
    ids = [im.split_id for im in imgs]
    for query in ("nested", "wide", "wide_retry"):
        plans = [plans_for(im, query) for im in imgs]
        times, retries, entries = [], 0, 0
        for step in range(a.warmup + a.steps):
            r = ctx.split_search(ids, plans)
            assert r[0].kernel_mask & ffi.KERNEL_HASHED_AGGS, hex(r[0].kernel_mask)
            if step >= a.warmup:
                times.append(r[0].gpu_time_us)
                retries += bool(r[0].kernel_mask & ffi.KERNEL_HASHED_AGGS_RETRY)
                entries = r[0].num_entries
        print(json.dumps({"workload": f"hashed_aggs_{query}", "splits": a.splits, "docs_per_split": a.docs,
                          "device_us_p50": float(np.percentile(times, 50)), "device_us_p99": float(np.percentile(times, 99)),
                          "calls": a.steps, "calls_with_retry": retries, "entries_split0": entries,
                          "gpu": gpu[0] if gpu else "unknown", "build_s": round(build_s, 1)}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
