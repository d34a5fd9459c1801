"""Wide aggregation requests (DESIGN.md §4.4, limits): one request of N aggregation nodes against the ceil(N / 8) requests a
client needed while a plan held at most 8 nodes, over --splits splits of --docs docs (32 x 3.125 M by default, the
split size of the config-5 corpus).

Corpus per split: `timestamp` (datetime over one day, seconds), `service` (20 values, Zipf), `status` (6 values),
`latency` (u64 < 2^20), `bytes` (u64 < 2^24) and f00..f11 (u64 of 4 to 20 bits).
Requests (match_all, no hits):
  * dashboard (10 nodes): terms(service) > date_histogram(1m) > {avg, min, max, percentiles of latency; sum, avg of
    bytes}, next to date_histogram(10m) and terms(status). Split: the latency half with the two top-level nodes
    (8 nodes), then the bytes half (4 nodes).
  * wide32 (32 nodes): terms(service) > 7 metrics, date_histogram(1h) > 7 metrics, 16 top-level metrics over
    f00..f11, latency and bytes. Split: four requests of 8 nodes.

For each form, the device time of a call (CUDA events, summed over the form's calls: split_search on the compiled
plans) p50 / p99, and the seam-A wall time (qwgpu_leaf_search on a LeafSearchRequest, host clock around the calls,
which return finished responses) p50 / p99. Prints one JSON line per request and form, with the card name and power
limit read in the same run. Nothing is written to the tree.

    python tools/bench_wide_aggs.py
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

from quickwit_b200 import ffi, proto, service, splitgen as S  # noqa: E402
from quickwit_b200.service import SearcherContext  # noqa: E402

T0 = 1_700_000_000
F = [f"f{i:02d}" for i in range(12)]
MAPPING = {"field_mappings": [{"name": "timestamp", "type": "datetime", "fast": True, "fast_precision": "seconds"}] +
           [{"name": n, "type": "u64", "fast": True} for n in ["service", "status", "latency", "bytes"] + F],
           "timestamp_field": "timestamp"}


def build(split_ord, n, seed):
    rng = np.random.default_rng(seed + split_ord)
    ts = (np.sort(rng.integers(0, 86_400, n)).astype(np.int64) + T0 + 86_400 * split_ord) * 10**9
    b = S._Builder(n)
    b.add_column("timestamp", ffi.COL_DATETIME, ffi.CARD_FULL, ts.view(np.uint64) ^ np.uint64(1 << 63), None)
    b.add_column("service", ffi.COL_U64, ffi.CARD_FULL, np.minimum(rng.zipf(1.5, n) - 1, 19).astype(np.uint64), None)
    b.add_column("status", ffi.COL_U64, ffi.CARD_FULL, rng.integers(0, 6, n, dtype=np.uint64), None)
    b.add_column("latency", ffi.COL_U64, ffi.CARD_FULL, rng.integers(0, 1 << 20, n, dtype=np.uint64), None)
    b.add_column("bytes", ffi.COL_U64, ffi.CARD_FULL, rng.integers(0, 1 << 24, n, dtype=np.uint64), None)
    for i, name in enumerate(F):
        b.add_column(name, ffi.COL_U64, ffi.CARD_FULL, rng.integers(0, 1 << (4 + i + i // 3), n, dtype=np.uint64), None)
    return b.finish(f"wide-{split_ord:03d}")


def _by_service(metrics, interval="1m"):
    return {"terms": {"field": "service"}, "aggs": {"per": {"date_histogram": {"field": "timestamp", "fixed_interval": interval},
                                                            "aggs": metrics}}}


LAT = {"lat_avg": {"avg": {"field": "latency"}}, "lat_min": {"min": {"field": "latency"}},
       "lat_max": {"max": {"field": "latency"}}, "lat_pct": {"percentiles": {"field": "latency"}}}
BYTES = {"bytes_sum": {"sum": {"field": "bytes"}}, "bytes_avg": {"avg": {"field": "bytes"}}}
OTHERS = {"over_time": {"date_histogram": {"field": "timestamp", "fixed_interval": "10m"}}, "by_status": {"terms": {"field": "status"}}}
KINDS = ("avg", "sum", "min", "max", "stats", "value_count")


def _metrics(fields, tag):
    return {f"{tag}_{f}_{k}": {k: {"field": f}} for f, k in zip(fields, KINDS * 4)}


REQUESTS = {
    "dashboard": ({"by_service": _by_service({**LAT, **BYTES}), **OTHERS},
                  [{"by_service": _by_service(LAT), **OTHERS}, {"by_service": _by_service(BYTES)}]),
    "wide32": ({"by_service": {"terms": {"field": "service"}, "aggs": _metrics(F[:7], "s")},
                "per_hour": {"date_histogram": {"field": "timestamp", "fixed_interval": "1h"}, "aggs": _metrics(F[5:12], "h")},
                **_metrics(F + ["latency", "bytes", "latency", "bytes"], "t")},
               [{"by_service": {"terms": {"field": "service"}, "aggs": _metrics(F[:7], "s")}},
                {"per_hour": {"date_histogram": {"field": "timestamp", "fixed_interval": "1h"}, "aggs": _metrics(F[5:12], "h")}},
                _metrics(F[:8], "t"), {k: v for k, v in _metrics(F + ["latency", "bytes", "latency", "bytes"], "t").items()
                                       if k not in _metrics(F[:8], "t")}]),
}


def _nodes(aggs):
    return sum(1 + _nodes(v.get("aggs", {})) for v in aggs.values())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--splits", type=int, default=32)
    ap.add_argument("--docs", type=int, default=3_125_000)
    ap.add_argument("--steps", type=int, default=20)
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
        print(json.dumps({"registered": i + 1}), flush=True)
    build_s = time.time() - t
    print(json.dumps({"corpus": f"{a.splits} x {a.docs}", "build_s": round(build_s, 1)}), flush=True)
    ids, dm = [im.split_id for im in imgs], json.dumps(MAPPING)
    offsets = [proto.enc_split_offsets(im.split_id, im.num_docs) for im in imgs]
    for name, (one, parts) in REQUESTS.items():
        assert _nodes(one) <= ffi.MAX_AGG_NODES and all(_nodes(p) <= 8 for p in parts), name
        for form, reqs in (("one_call", [one]), (f"{len(parts)}_calls", parts)):
            sreqs = [proto.enc_search_request(json.dumps({"type": "match_all"}), max_hits=0, aggregation_request=json.dumps(r))
                     for r in reqs]
            plans = [[service.compile_plan(im, sr, dm) for im in imgs] for sr in sreqs]
            lreqs = [proto.enc_leaf_search_request(sr, offsets, dm) for sr in sreqs]
            dev, wall = [], []
            for step in range(a.warmup + a.steps):
                d = 0.0
                for p in plans:
                    r = ctx.split_search(ids, p)
                    assert r[0].kernel_mask & ffi.KERNEL_WINDOW and not r[0].kernel_mask & ffi.KERNEL_AGGSCAN, hex(r[0].kernel_mask)
                    d += r[0].gpu_time_us
                t0 = time.perf_counter()
                for lr in lreqs:
                    resp = proto.dec_leaf_search_response(ctx.leaf_search(lr))
                    assert not resp.get("failed_splits"), resp.get("failed_splits")
                w = (time.perf_counter() - t0) * 1e6
                if step >= a.warmup:
                    dev.append(d)
                    wall.append(w)
            print(json.dumps({"workload": f"wide_aggs_{name}", "form": form, "nodes": [_nodes(r) for r in reqs],
                              "splits": a.splits, "docs_per_split": a.docs,
                              "device_us_p50": round(float(np.percentile(dev, 50)), 1),
                              "device_us_p99": round(float(np.percentile(dev, 99)), 1),
                              "seam_a_us_p50": round(float(np.percentile(wall, 50)), 1),
                              "seam_a_us_p99": round(float(np.percentile(wall, 99)), 1),
                              "calls": a.steps, "gpu": gpu[0] if gpu else "unknown", "build_s": round(build_s, 1)}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
