#!/usr/bin/env python
"""A dashboard refresh loop over the partial-result cache (DESIGN.md §7.1), cache off against cache on.

Corpus: bench.py's config-5 corpus (32 splits x 3.125 M docs, one day of timestamps per split). Request: a time
window of 16 days that slides by 1/32 of its span (half a day) per call; `date_histogram(1m) > {avg, max}` plus the
top 100 hits by timestamp. The synthetic corpus has no latency column: tenant_id stands in for it.

Two contexts hold the same splits, one with the cache off and one with it on, and each step calls both, alternating
which goes first. Reported per mode: seam-A wall time (host clock around the synchronous call) and device time (the
sum of the response's per-split cpu_search_microsecs, the split shares of the batch's device time) at p50 / p99. Cold
calls (the cache on but empty) against cache-off calls give the cost of building and storing every split's own
response. Every cached response is checked against the uncached one.

    python tools/bench_leaf_cache.py [--splits 32] [--docs-per-split 3125000] [--calls 32] --out leaf_cache.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

T0 = 1_700_000_000
DAY = 86_400
AGGS = {"per_minute": {"date_histogram": {"field": "timestamp", "fixed_interval": "1m"},
                       "aggs": {"avg_latency": {"avg": {"field": "tenant_id"}}, "max_latency": {"max": {"field": "tenant_id"}}}}}


def pct(v, p):
    v = sorted(v)
    return v[min(len(v) - 1, int(round(p / 100 * (len(v) - 1))))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--splits", type=int, default=32)
    ap.add_argument("--docs-per-split", type=int, default=3_125_000)
    ap.add_argument("--calls", type=int, default=32, help="refreshes per pass (the window must stay inside the corpus)")
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    from quickwit_b200 import proto
    from quickwit_b200.service import SearcherContext
    span = DAY * a.splits // 2
    step = span // 32
    if DAY // 4 + (a.calls - 1) * step + span > DAY * a.splits:
        sys.exit("--calls too large: the window would leave the corpus")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    imgs = bench.build_splits(0, a.splits, a.docs_per_split, threads=min(os.cpu_count() or 1, 32), msg_vocab=bench.MSG_VOCAB)
    dm = json.dumps(bench.SYNTH_MAPPING)
    offsets = [proto.enc_split_offsets(im.split_id, im.num_docs, timestamp_start=T0 + DAY * i, timestamp_end=T0 + DAY * (i + 1) - 1)
               for i, im in enumerate(imgs)]

    def request(k):
        start = T0 + DAY // 4 + k * step
        sreq = proto.enc_search_request(json.dumps({"type": "match_all"}), max_hits=100, sort_fields=[("timestamp", proto.DESC)],
                                        aggregation_request=json.dumps(AGGS), start_timestamp=start, end_timestamp=start + span)
        return proto.enc_leaf_search_request(sreq, offsets, dm)

    off, on = SearcherContext(0), SearcherContext(0)
    for im in imgs:
        off.register_split(im)
        on.register_split(im)
    on.set_leaf_cache_budget(64 << 20)  # Quickwit's default searcher.partial_request_cache_capacity

    def call(ctx, req):
        t = time.perf_counter()
        resp = ctx.leaf_search(req)
        wall = (time.perf_counter() - t) * 1e6
        d = proto.dec_leaf_search_response(resp)
        rs = d["resource_stats"] or {}
        dev = (rs.get("split_resources_sum") or {}).get("cpu_search_microsecs", 0)
        same = {k: d[k] for k in ("num_hits", "partial_hits", "failed_splits", "num_attempted_splits", "num_successful_splits")}
        return wall, dev, rs.get("partial_result_cache_num_splits", 0), same, d["intermediate_aggregation_result"]

    reqs = [request(k) for k in range(a.calls)]
    for r in reqs[:2]:  # warm-up: modules, call slots, host allocations
        call(off, r)
        call(on, r)
    # cold calls: the cache on but emptied before every call, against the cache off
    cold = {"off": [], "on": []}
    for k, r in enumerate(reqs[: min(8, a.calls)]):
        on.set_leaf_cache_budget(0)
        on.set_leaf_cache_budget(64 << 20)
        order = (("off", off), ("on", on)) if k % 2 == 0 else (("on", on), ("off", off))
        for name, ctx in order:
            cold[name].append(call(ctx, r)[0])
    # the refresh loop
    res = {"off": {"wall": [], "dev": []}, "on": {"wall": [], "dev": [], "cached_splits": []}}
    mismatches = 0
    from quickwit_b200 import service
    for p in range(a.passes):
        on.set_leaf_cache_budget(0)
        on.set_leaf_cache_budget(64 << 20)
        for k, r in enumerate(reqs):
            order = (("off", off), ("on", on)) if (k + p) % 2 == 0 else (("on", on), ("off", off))
            out = {}
            for name, ctx in order:
                out[name] = call(ctx, r)
            for name in ("off", "on"):
                res[name]["wall"].append(out[name][0])
                res[name]["dev"].append(out[name][1])
            res["on"]["cached_splits"].append(out["on"][2])
            fin = [service.finalize_aggregation(json.dumps(AGGS), out[n][4] or b"") for n in ("off", "on")]
            if out["off"][3] != out["on"][3] or fin[0] != fin[1]:
                mismatches += 1
    summary = {"gpu": gpu, "splits": a.splits, "docs_per_split": a.docs_per_split, "calls": a.calls * a.passes,
               "window_days": span / DAY, "step_days": step / DAY, "mismatches": mismatches,
               "cold_wall_us_p50": {n: pct(v, 50) for n, v in cold.items()},
               "cold_wall_us": cold}
    for name in ("off", "on"):
        for m in ("wall", "dev"):
            summary[f"{name}_{m}_us_p50"] = pct(res[name][m], 50)
            summary[f"{name}_{m}_us_p99"] = pct(res[name][m], 99)
    summary["on_cached_splits_mean"] = sum(res["on"]["cached_splits"]) / len(res["on"]["cached_splits"])
    on.close()
    off.close()
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    json.dump(dict(summary, raw=res), open(a.out, "w"), indent=1)
    print(json.dumps(summary, indent=1))
    if mismatches:
        sys.exit(f"{mismatches} cached responses differ from the uncached ones")


if __name__ == "__main__":
    main()
