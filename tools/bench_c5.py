#!/usr/bin/env python
"""BASELINE config 5's shape on one GPU at several concurrency levels (bench.py's config5_mixed block alone).

    python tools/bench_c5.py [--splits 32] [--docs-per-split 3125000] [--concurrency 1,8,64] --out c5.json
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--splits", type=int, default=32)
    ap.add_argument("--docs-per-split", type=int, default=3_125_000)
    ap.add_argument("--concurrency", default="1,8,64")
    ap.add_argument("--out", required=True)
    ap.add_argument("--announce", action="store_true", help="print the query type before every call (pair with QWGPU_TRACE=1)")
    a = ap.parse_args()
    import torch
    from quickwit_b200.service import SearcherContext
    torch.cuda.set_device(0)
    imgs = bench.build_splits(0, a.splits, a.docs_per_split, threads=min(os.cpu_count() or 1, 32), msg_vocab=bench.MSG_VOCAB)
    ctx = SearcherContext(0)
    for im in imgs:
        ctx.register_split(im)
    peak = bench.DATASHEET_HBM_GBS
    try:
        peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))).get("hbm_gbs", peak))
    except Exception:
        pass
    rows = []
    for c in [int(x) for x in a.concurrency.split(",")]:
        r = bench.config5_mixed(ctx, imgs, peak, 1, concurrency=c, queries_per_thread=max(6, 96 // c), announce=a.announce)
        rows.append(r)
        print(json.dumps({"concurrency": c, "cores": os.cpu_count(), "qps": r["qps"], "latency_ms": r["latency_ms"], "hbm_frac": r["hbm"]["frac"]}), flush=True)
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    json.dump(rows, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
