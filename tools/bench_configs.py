#!/usr/bin/env python
"""Latency of the BASELINE.json configs C1-C4 (plus a few sort/filter variants) on one GPU.

Not the headline bench (that is bench.py = C2); this writes a per-config table: device time
through qwgpu_split_search (seam C), wall time through qwgpu_leaf_search (protobuf in/out), and the oracle port on a sample of the splits for scale.

    python tools/bench_configs.py [--splits 32] [--docs-per-split 3125000] [--reps 20] --out configs.json
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402  (RawSearch, build_splits)

T0 = 1_700_000_000
MAPPING = {"field_mappings": [{"name": "body", "type": "text", "record": "freq", "fieldnorms": True},
                              {"name": "severity_text", "type": "text", "tokenizer": "raw", "fast": True},
                              {"name": "timestamp", "type": "datetime", "fast": True, "fast_precision": "seconds"},
                              {"name": "tenant_id", "type": "u64", "fast": True}], "timestamp_field": "timestamp"}


def term(f, v):
    return {"type": "term", "field": f, "value": v}


def configs(n_splits):
    or10 = {"type": "bool", "should": [term("body", f"t{i}") for i in range(10)]}
    span = 86_400 * n_splits
    return [
        ("C1 term(severity_text:ERROR) top-10 by doc id", term("severity_text", "ERROR"), dict(max_hits=10)),
        ("C1b term(body:t0, 20% of docs) top-10 by BM25", term("body", "t0"), dict(max_hits=10, sort_fields=[("_score", 1)])),
        ("C2 10-term OR, BM25 top-1000", or10, dict(max_hits=1000, sort_fields=[("_score", 1)])),
        ("C2b 10-term OR, count only", or10, dict(max_hits=0)),
        # experiments on the clause chain of the BM25-union pipeline: only the 4 dense terms / only the 6 sparse ones
        ("X2d 4 dense terms OR, BM25 top-1000", {"type": "bool", "should": [term("body", f"t{i}") for i in range(4)]}, dict(max_hits=1000, sort_fields=[("_score", 1)])),
        ("X2s 6 sparse terms OR, BM25 top-1000", {"type": "bool", "should": [term("body", f"t{i}") for i in range(4, 10)]}, dict(max_hits=1000, sort_fields=[("_score", 1)])),
        ("X2t 2 dense terms OR, BM25 top-1000", {"type": "bool", "should": [term("body", f"t{i}") for i in range(2)]}, dict(max_hits=1000, sort_fields=[("_score", 1)])),
        ("C3 term AND timestamp range (half the span), top-1000 by timestamp desc", {"type": "bool", "must": [term("body", "t2")]},
         dict(max_hits=1000, sort_fields=[("timestamp", 1)], start_timestamp=T0 + span // 4, end_timestamp=T0 + 3 * span // 4)),
        ("C3b 2-term AND NOT third, top-100 by (tenant_id asc, timestamp desc)",
         {"type": "bool", "must": [term("body", "t0"), term("body", "t1")], "must_not": [term("body", "t4")]},
         dict(max_hits=100, sort_fields=[("tenant_id", 0), ("timestamp", 1)])),
        ("C4 match_all, terms(severity_text) + date_histogram(1h)", {"type": "match_all"},
         dict(max_hits=0, aggs={"by_sev": {"terms": {"field": "severity_text"}},
                                "over_time": {"date_histogram": {"field": "timestamp", "fixed_interval": "1h"}}})),
        ("C4b 10-term OR, terms(tenant_id) > stats(timestamp)", or10,
         dict(max_hits=0, aggs={"tenants": {"terms": {"field": "tenant_id", "size": 10}, "aggs": {"ts": {"stats": {"field": "timestamp"}}}}})),
    ]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--splits", type=int, default=32)
    ap.add_argument("--docs-per-split", type=int, default=3_125_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--cpu-splits", type=int, default=8)
    ap.add_argument("--only", default="", help="run only configs whose name starts with this prefix (e.g. C4)")
    ap.add_argument("--no-oracle", action="store_true")
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    import torch
    from quickwit_b200 import proto, service
    from quickwit_b200.service import SearcherContext
    from oracle import oracle as O
    torch.cuda.set_device(0)
    cores = os.cpu_count() or 1
    imgs = bench.build_splits(0, a.splits, a.docs_per_split, threads=min(cores, 32))
    ctx = SearcherContext(0)
    for im in imgs:
        ctx.register_split(im)
    ids = [im.split_id for im in imgs]
    dm = json.dumps(MAPPING)
    offsets = [proto.enc_split_offsets(im.split_id, im.num_docs) for im in imgs]
    rows = []
    for name, ast, kw in configs(a.splits):
        if a.only and not any(name.startswith(o + " ") for o in a.only.split(",")):
            continue
        kw = dict(kw)
        aggs = kw.pop("aggs", None)
        sreq = proto.enc_search_request(json.dumps(ast), aggregation_request=json.dumps(aggs) if aggs else None, **kw)
        lreq = proto.enc_leaf_search_request(sreq, offsets, dm)
        plans = [service.compile_plan(im, sreq, dm) for im in imgs]
        rs = bench.RawSearch(ctx, ids, plans)
        for _ in range(3):
            rs.run(); rs.free()
        gpu_us = main_us = 0.0
        for _ in range(a.reps):
            r = rs.run(); rs.free()
            gpu_us += r["gpu_us"]; main_us += r["main_us"]
        for _ in range(3):
            resp = ctx.leaf_search(lreq)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.reps):
            resp = ctx.leaf_search(lreq)
        wall = (time.perf_counter() - t0) / a.reps
        dec = proto.dec_leaf_search_response(resp)
        # oracle port on a sample of the splits, one split per thread
        ns = min(a.cpu_splits, a.splits)
        def one(i):
            return O.split_search(imgs[i], plans[i]).num_hits
        cpu = 0.0
        if not a.no_oracle:
            with ThreadPoolExecutor(max_workers=ns) as ex:
                list(ex.map(one, range(ns)))
                t0 = time.perf_counter()
                list(ex.map(one, range(ns)))
                cpu = time.perf_counter() - t0
        docs = a.splits * a.docs_per_split
        row = {"config": name, "num_hits": dec["num_hits"], "partial_hits": len(dec["partial_hits"]),
               "device_us": gpu_us / a.reps, "k_window_collect_us": main_us / a.reps, "launches": r["launches"],
               "algorithmic_mb": r["alg_bytes"] / 1e6, "postings_scored": r["postings"], "exact_fallbacks": r["fallbacks"],
               "algorithmic_gbs_device": r["alg_bytes"] / (gpu_us / a.reps) / 1e3 if gpu_us else None,
               "leaf_search_wall_us": 1e6 * wall, "docs": docs,
               "oracle_us_scaled": 1e6 * cpu * a.splits / ns, "oracle_threads": ns}
        rows.append(row)
        print(json.dumps(row), flush=True)
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        json.dump({"splits": a.splits, "docs_per_split": a.docs_per_split, "reps": a.reps, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
