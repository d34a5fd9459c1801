"""`missing` on the stats family (DESIGN.md §4.4, stats-family `missing`): device time of the latency dashboard panels
with `missing` against the same requests without it, over --splits splits of --docs log docs (32 x 3.125 M by
default, the size of the config-5 corpus).

Corpus per split: a datetime column over one day at second precision and `latency` (u64 < 2^20), absent on about
30 % of the docs and holding two or three values on about 10 % (a multi-valued column, so every request takes the
generic dense walk).
Queries (match_all, no hits, one call over every split):
  * date_histogram(1h) > {avg, min, max}(latency, missing: 0)   vs   the same without `missing`;
  * stats(latency, missing: -1)                                  vs   stats(latency).

Prints one JSON line per query: device time p50 / p99 of the call (CUDA events), the kernel path, the cells of split
0, and the card name and power limit read in the same run. Nothing is written to the tree.

    python tools/bench_metric_missing.py
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
    per = rng.choice(np.array([0, 1, 2, 3], dtype=np.uint32), size=n, p=[0.3, 0.6, 0.05, 0.05])
    start = np.zeros(n + 1, dtype=np.uint32)
    np.cumsum(per, out=start[1:])
    b = S._Builder(n)
    b.add_column("timestamp", ffi.COL_DATETIME, ffi.CARD_FULL, ts.view(np.uint64) ^ np.uint64(1 << 63), None)
    b.add_column("latency", ffi.COL_U64, ffi.CARD_MULTI, rng.integers(0, 1 << 20, int(start[-1]), dtype=np.uint64), start)
    return b.finish(f"mm-{split_ord:03d}")


def plans_for(img, query):
    ts, lat = img.column_ord("timestamp"), img.column_ord("latency")
    with_missing = not query.endswith("_plain")
    if query.startswith("date_histogram"):
        h = img.columns()[ts]
        base, top = S.u64_to_i64(h.min_value) // HOUR_NS, S.u64_to_i64(h.max_value) // HOUR_NS
        # avg, min and max of one field are three stats nodes, as the request compiles them
        metrics = [P.stats(lat, 0.0 if with_missing else None) for _ in range(3)]
        aggs = [P.Agg(ffi.AGG_HISTOGRAM, column=ts, num_buckets=int(top - base + 1), interval=float(HOUR_NS),
                      base_pos=int(base), children=metrics)]
    else:
        aggs = [P.stats(lat, -1.0 if with_missing else None)]
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
    queries = ("date_histogram_avg_min_max", "date_histogram_avg_min_max_plain", "stats", "stats_plain")
    plans = {q: [plans_for(im, q) for im in imgs] for q in queries}
    times = {q: [] for q in queries}
    info = {}
    for step in range(a.warmup + a.steps):
        for q in queries:  # alternated, so that drift on the shared machine hits every query alike
            r = ctx.split_search(ids, plans[q])
            if step >= a.warmup:
                times[q].append(r[0].gpu_time_us)
            info[q] = (r[0].kernel_mask, len(r[0].cells))
    for q in queries:
        mask, cells = info[q]
        print(json.dumps({"workload": q, "splits": a.splits, "docs_per_split": a.docs,
                          "device_us_p50": float(np.percentile(times[q], 50)), "device_us_p99": float(np.percentile(times[q], 99)),
                          "calls": a.steps, "kernel_mask": mask, "cells_split0": cells,
                          "gpu": gpu[0] if gpu else "unknown", "build_s": round(build_s, 1)}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
