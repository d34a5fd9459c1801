"""Deep top-K: qwgpu_leaf_search latency at K = max_hits from 1000 to 20 000 on the bench's index (32 splits x 3.125 M
docs, bench.py's generator), for the C2 query (BM25 10-term OR by `_score`) and a column sort (term body:t2 by
timestamp desc). K > 4096 takes the deep selection path (deep_select_kernel.cuh).

Per (query, K): p50 / p99 of the wall time of --steps qwgpu_leaf_search calls (host protobuf bytes in and out, every
split's list merged on the device), the device time p50 and kernel launches of the same plans through seam C
(qwgpu_split_search, no merge), and the bytes copied back per leaf call, computed from the output layout (per split a
256-byte-aligned header + aggregation region, then the merged record of 64 + K x 40 bytes). Prints the card's name and
power limit first, then one JSON line per row. Nothing is written to the tree.

    python tools/bench_deep_topk.py
    python tools/bench_deep_topk.py --splits 4 --docs 200000 --steps 3   # a quick run
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
    ap.add_argument("--splits", type=int, default=32)
    ap.add_argument("--docs", type=int, default=3_125_000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ks", default="1000,4096,4097,10000,20000")
    a = ap.parse_args()
    import bench
    from bench_phrase_prefix import card
    from quickwit_b200 import proto, service
    from quickwit_b200.service import SearcherContext

    print(json.dumps({"card": card()}), flush=True)
    ctx = SearcherContext(0)
    ctx.set_max_hits(20_000)
    t = time.time()
    imgs = bench.build_splits(0, a.splits, a.docs, threads=min(os.cpu_count() or 1, 32))
    for img in imgs:
        ctx.register_split(img)
    build_s = time.time() - t
    dm = json.dumps(bench.SYNTH_MAPPING)
    ids = [im.split_id for im in imgs]
    offsets = [proto.enc_split_offsets(im.split_id, im.num_docs) for im in imgs]
    queries = {
        "c2_bm25_or10": ({"type": "bool", "should": [{"type": "term", "field": "body", "value": f"t{i}"} for i in range(10)]},
                         [("_score", proto.DESC)]),
        "term_by_timestamp": ({"type": "term", "field": "body", "value": "t2"}, [("timestamp", proto.DESC)]),
    }
    for name, (ast, sort) in queries.items():
        for K in [int(x) for x in a.ks.split(",")]:
            sreq = proto.enc_search_request(json.dumps(ast), max_hits=K, sort_fields=sort)
            lreq = proto.enc_leaf_search_request(sreq, offsets, dm)
            plans = [service.compile_plan(im, sreq, dm) for im in imgs]
            dev, launches, mask, fallbacks = [], 0, 0, 0
            for step in range(a.warmup + a.steps):
                r = ctx.split_search(ids, plans)
                if step >= a.warmup:
                    dev.append(r[0].gpu_time_us)
                launches, mask, fallbacks = r[0].num_kernel_launches, r[0].kernel_mask, max(fallbacks, r[0].exact_fallbacks)
            lat = []
            for step in range(a.warmup + a.steps):
                t0 = time.perf_counter()
                resp = ctx.leaf_search(lreq)
                if step >= a.warmup:
                    lat.append(time.perf_counter() - t0)
            dec = proto.dec_leaf_search_response(resp)
            assert len(dec["partial_hits"]) == min(K, dec["num_hits"])
            d2h = a.splits * 256 + 64 + K * 40
            print(json.dumps({"query": name, "k": K, "splits": a.splits, "docs_per_split": a.docs, "calls": a.steps,
                              "leaf_search_p50_ms": round(1e3 * float(np.percentile(lat, 50)), 3),
                              "leaf_search_p99_ms": round(1e3 * float(np.percentile(lat, 99)), 3),
                              "seam_c_device_p50_us": round(float(np.percentile(dev, 50)), 1), "seam_c_launches": launches,
                              "deep_select": bool(mask & 2048), "exact_fallbacks": fallbacks,
                              "leaf_d2h_bytes": d2h, "num_hits": dec["num_hits"], "build_s": round(build_s, 1)}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
