"""Phrase-prefix queries on the GPU: device time of the PHRASE_PREFIX node against the OR of one plain phrase per
expansion, over the config-5 shaped corpus (synthetic splits with the positions field `msg`, vocabulary w0..w63).

Queries: `w0 w1*` (frequent exact term), `w40 w1*` (rare exact term), `w1 w2 w3*`, the single-token `w1*` (its set
filter of terms) and the plain phrase `w1 w2`. For each, device time p50 / p99 over --steps calls of
qwgpu_split_search over every split (CUDA events), and for the multi-token prefixes the same for the OR-of-phrases plan
with a check that both return the same hits. Prints the card's name and power limit first, then one JSON line per
query. Nothing is written to the tree.

    python tools/bench_phrase_prefix.py
    python tools/bench_phrase_prefix.py --root OTHER_TREE --only plain   # the plain phrase on another build
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # (the timings stand without it)
        return {"gpu": "unknown", "error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--splits", type=int, default=32)
    ap.add_argument("--docs", type=int, default=3_125_000)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--root", default=ROOT, help="tree to import quickwit_b200 from (to time another build)")
    ap.add_argument("--only", choices=["all", "plain"], default="all")
    a = ap.parse_args()
    sys.path.insert(0, a.root)
    from quickwit_b200 import ffi, plan as P, splitgen as S
    from quickwit_b200.service import SearcherContext

    print(json.dumps({"card": card(), "root": "head" if os.path.abspath(a.root) == ROOT else "other"}), flush=True)
    ctx = SearcherContext(0)
    t = time.time()
    imgs = []
    for i in range(a.splits):
        img = S.synth_split(a.docs, i, [0.2, 0.05], split_id=f"c5pp-{i:03d}", msg_vocab=64)
        ctx.register_split(img)
        imgs.append(img)
    build_s = time.time() - t
    ids = [im.split_id for im in imgs]
    sort = [(ffi.SORT_DOCID, ffi.ORDER_DESC, ffi.ABSENT)]

    def timed(plans):
        times, r = [], None
        for step in range(a.warmup + a.steps):
            r = ctx.split_search(ids, plans)
            if step >= a.warmup:
                times.append(r[0].gpu_time_us)
        return {"p50_us": float(np.percentile(times, 50)), "p99_us": float(np.percentile(times, 99)),
                "num_hits": sum(x.num_hits for x in r)}, [(x.num_hits, x.hits) for x in r]

    queries = [("w1 w2", None)] if a.only == "plain" else [("w0 w1*", 50), ("w40 w1*", 50), ("w1 w2 w3*", 50), ("w1*", 50), ("w1 w2", None)]
    for q, m in queries:
        tokens = q.rstrip("*").split()
        row = {"query": q, "splits": a.splits, "docs_per_split": a.docs, "k": a.k, "calls": a.steps, "build_s": round(build_s, 1)}
        if m is None:
            row["phrase"], _ = timed([P.make_plan(P.phrase(im, "msg", tokens), a.k, sort) for im in imgs])
        else:
            nodes = [P.phrase_prefix(im, "msg", tokens, m) for im in imgs]
            row["expansions_split0"] = len(P.prefix_expansions(imgs[0], "msg", tokens[-1], m))
            row["phrase_prefix"], out = timed([P.make_plan(n, a.k, sort) for n in nodes])
            if len(tokens) > 1:
                row["or_of_phrases"], out_or = timed([P.make_plan(P.phrase_prefix_as_phrases(n), a.k, sort) for n in nodes])
                row["same_output"] = out == out_or
        print(json.dumps(row), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
