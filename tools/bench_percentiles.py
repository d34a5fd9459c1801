"""Percentiles aggregations on the GPU (DESIGN.md §4.4, percentiles): device time of the latency-percentile dashboard
query against the same tree with `stats` in place of `percentiles`, over --splits splits of --docs log docs (32 x
3.125 M by default, the size of the config-5 corpus).

Corpus per split: a datetime column over one day at second precision and `latency` (u64 < 2^20), as in
tools/bench_nested_aggs.py.
Queries (match_all, no hits, one call over every split):
  * date_histogram(1h) > percentiles(latency)   vs   date_histogram(1h) > stats(latency);
  * percentiles(latency)                        vs   stats(latency).

Prints one JSON line per query: device time p50 / p99 of the call (CUDA events), the kernel path, the number of
entries of split 0, and the card name and power limit read in the same run. Nothing is written to the tree.

    python tools/bench_percentiles.py
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

from quickwit_b200 import ffi, plan as P, service, splitgen as S  # noqa: E402
from quickwit_b200.service import SearcherContext  # noqa: E402

T0 = 1_700_000_000
HOUR_NS = 3600 * 10**9


def build(split_ord, n, seed):
    rng = np.random.default_rng(seed + split_ord)
    ts = np.sort(rng.integers(0, 86_400, n)).astype(np.int64) * 10**9 + (T0 + 86_400 * split_ord) * 10**9
    b = S._Builder(n)
    b.add_column("timestamp", ffi.COL_DATETIME, ffi.CARD_FULL, ts.view(np.uint64) ^ np.uint64(1 << 63), None)
    b.add_column("latency", ffi.COL_U64, ffi.CARD_FULL, rng.integers(0, 1 << 20, n, dtype=np.uint64), None)
    return b.finish(f"pct-{split_ord:03d}")


def plans_for(img, query):
    ts, lat = img.column_ord("timestamp"), img.column_ord("latency")
    if query.endswith("percentiles"):
        metric = P.percentiles(lat, len(service.percentiles_table(img, lat)[1]))
    else:
        metric = P.Agg(ffi.AGG_STATS, column=lat)
    if query.startswith("date_histogram"):
        h = img.columns()[ts]
        base, top = S.u64_to_i64(h.min_value) // HOUR_NS, S.u64_to_i64(h.max_value) // HOUR_NS
        aggs = [P.Agg(ffi.AGG_HISTOGRAM, column=ts, num_buckets=int(top - base + 1), interval=float(HOUR_NS),
                      base_pos=int(base), children=[metric])]
    else:
        aggs = [metric]
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
    queries = ("date_histogram_percentiles", "date_histogram_stats", "percentiles", "stats")
    plans = {q: [plans_for(im, q) for im in imgs] for q in queries}
    times = {q: [] for q in queries}
    info = {}
    for step in range(a.warmup + a.steps):
        for q in queries:  # alternated, so that drift on the shared machine hits every query alike
            r = ctx.split_search(ids, plans[q])
            if step >= a.warmup:
                times[q].append(r[0].gpu_time_us)
            info[q] = (r[0].kernel_mask, r[0].num_entries, len(r[0].cells))
    for q in queries:
        mask, entries, cells = info[q]
        print(json.dumps({"workload": q, "splits": a.splits, "docs_per_split": a.docs,
                          "device_us_p50": float(np.percentile(times[q], 50)), "device_us_p99": float(np.percentile(times[q], 99)),
                          "calls": a.steps, "kernel_mask": mask, "entries_split0": entries, "cells_split0": cells,
                          "gpu": gpu[0] if gpu else "unknown", "build_s": round(build_s, 1)}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
