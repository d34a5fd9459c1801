"""Leaf requests over many splits: device time per qwgpu_leaf_search call and the share of the device merge
(k_merge_prep + k_merge) at n = 32, 65, 128 and 300 splits for K = 10, 1000 and 20 000.

Above 64 lists k_merge_prep does not prune, so every hit of every list takes part in k_merge: each warp ranks one hit
by a binary search in every other list, about n^2 * K * log K probes. This tool measures what that costs.

The splits are --bases synthetic splits of --docs docs (bench.py's generator), each registered under n / bases ids.
Two queries: a BM25 OR of four terms by `_score` (k_union) and one term by timestamp desc (a column sort). Per row:
- the device time of every kernel of a leaf call and of the merge kernels, from torch.profiler's CUDA activity records
  over --steps calls (a separate run of the same calls, after the timed one);
- the wall time p50 of --steps leaf calls, profiler off;
- the device time p50 of the same plans through seam C (qwgpu_split_search, which does not merge).
Prints the card's name and power limit first, then one JSON line per row. Nothing is written to the tree.

    python tools/bench_many_splits.py
    python tools/bench_many_splits.py --ns 32 --ks 10 --docs 20000 --steps 2   # a quick run
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ns", default="32,65,128,300")
    ap.add_argument("--ks", default="10,1000,20000")
    ap.add_argument("--bases", type=int, default=8)
    ap.add_argument("--docs", type=int, default=250_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    from bench_phrase_prefix import card
    from quickwit_b200 import proto, service, splitgen as S
    from quickwit_b200.service import SearcherContext

    print(json.dumps({"card": card()}), flush=True)
    torch.cuda.init()
    ctx = SearcherContext(0)
    ctx.set_max_hits(20_000)
    bases = [S.synth_split(a.docs, i, bench.FRACS,
                           split_id=f"base-{i}", ts_start_secs=1_700_000_000 + 86_400 * i) for i in range(a.bases)]
    dm = json.dumps(bench.SYNTH_MAPPING)
    queries = {
        "bm25_or4": ({"type": "bool", "should": [{"type": "term", "field": "body", "value": f"t{i}"} for i in range(4)]},
                     [("_score", proto.DESC)]),
        "term_by_timestamp": ({"type": "term", "field": "body", "value": "t1"}, [("timestamp", proto.DESC)]),
    }
    registered = set()
    for n in [int(x) for x in a.ns.split(",")]:
        ids = [f"s-{i:04d}" for i in range(n)]
        for i, sid in enumerate(ids):
            if sid not in registered:
                ctx.register_split(bases[i % a.bases], split_id=sid)
                registered.add(sid)
        imgs = [S.SplitImage(bases[i % a.bases].array, sid) for i, sid in enumerate(ids)]
        offsets = [proto.enc_split_offsets(sid, a.docs) for sid in ids]
        for name, (ast, sort) in queries.items():
            for K in [int(x) for x in a.ks.split(",")]:
                sreq = proto.enc_search_request(json.dumps(ast), max_hits=K, sort_fields=sort)
                lreq = proto.enc_leaf_search_request(sreq, offsets, dm)
                plans = [service.compile_plan(im, sreq, dm) for im in imgs]
                dev = []
                for step in range(a.warmup + a.steps):
                    r = ctx.split_search(ids, plans)
                    if step >= a.warmup:
                        dev.append(r[0].gpu_time_us)
                lat = []
                for step in range(a.warmup + a.steps):
                    t0 = time.perf_counter()
                    resp = ctx.leaf_search(lreq)
                    if step >= a.warmup:
                        lat.append(time.perf_counter() - t0)
                dec = proto.dec_leaf_search_response(resp)
                assert len(dec["partial_hits"]) == min(K, dec["num_hits"]) and not dec["failed_splits"]
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(a.steps):
                        ctx.leaf_search(lreq)
                    torch.cuda.synchronize()
                total = merge = 0.0
                for ev in prof.events():
                    if ev.device_type == torch.autograd.DeviceType.CUDA and "k_" in ev.name:
                        us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
                        total += us
                        if "k_merge" in ev.name:
                            merge += us
                print(json.dumps({"query": name, "splits": n, "k": K, "docs_per_split": a.docs, "calls": a.steps,
                                  "leaf_device_us_per_call": round(total / a.steps, 1),
                                  "merge_device_us_per_call": round(merge / a.steps, 1),
                                  "merge_share": round(merge / total, 3) if total else None,
                                  "leaf_wall_p50_ms": round(1e3 * float(np.percentile(lat, 50)), 3),
                                  "seam_c_device_p50_us": round(float(np.percentile(dev, 50)), 1),
                                  "num_hits": dec["num_hits"]}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
