"""`ip` fields against u64 fields (DESIGN.md §4.10): device time of two match-all shapes over --splits splits of --docs
docs (32 x 3.125 M by default), each next to the same shape over a u64 column.

Corpus per split: `client_ip`, a fast `ip` field with 2^16 distinct IPv4 addresses (a QW_COL_IP column: ordinals into
the split's sorted address dictionary), and `client_u64`, a fast u64 field with 2^16 distinct values spread over the
u64 range (k << 40 for address k), drawn for the same docs. Both are 16-bit packed, so the device reads the same
bytes for either.
Queries (one call over every split, compiled from protobuf requests like a leaf search):
  * range: `client_ip:[10.0.0.0 TO <address 32767>]` (about half the docs), top 10 by doc id; and the u64 twin;
  * terms: terms(client_ip, size 10) with no hits; and terms(client_u64, size 10).

Prints one JSON line per shape: device time p50 / p99 of the call (CUDA events), and the card name and power limit
read in the same run. Nothing is written to the tree.

    python tools/bench_ip.py
"""
import argparse
import ipaddress
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

N_ADDR = 1 << 16
BASE = int(ipaddress.IPv4Address("10.0.0.0"))
DM = json.dumps({"field_mappings": [{"name": "client_ip", "type": "ip", "indexed": False, "fast": True},
                                    {"name": "client_u64", "type": "u64", "fast": True}]})


def address(k):
    return str(ipaddress.IPv4Address(BASE + 251 * k))


def build(split_ord, n, seed):
    rng = np.random.default_rng(seed + split_ord)
    k = rng.integers(0, N_ADDR, n, dtype=np.uint64)
    present = np.unique(k)
    ords = np.searchsorted(present, k).astype(np.uint64)
    dictionary = [S.parse_ip(address(int(x))) for x in present]
    b = S._Builder(n)
    b.add_column("client_ip", ffi.COL_IP, ffi.CARD_FULL, ords, None, dictionary)
    b.add_column("client_u64", ffi.COL_U64, ffi.CARD_FULL, k << np.uint64(40), None)
    return b.finish(f"ip-{split_ord:03d}")


def request(shape, field):
    if shape == "range":
        hi = address(N_ADDR // 2 - 1) if field == "client_ip" else str((N_ADDR // 2 - 1) << 40)
        lo = address(0) if field == "client_ip" else "0"
        ast = {"type": "range", "field": field, "lower_bound": {"Included": lo}, "upper_bound": {"Included": hi}}
        return proto.enc_search_request(json.dumps(ast), max_hits=10, sort_fields=[("_doc", 1)])
    aggs = {"top": {"terms": {"field": field, "size": 10}}}
    return proto.enc_search_request(json.dumps({"type": "match_all"}), max_hits=0, aggregation_request=json.dumps(aggs))


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
        img = build(i, a.docs, 0x1A)
        ctx.register_split(img)
        imgs.append(img)
    build_s = time.time() - t
    ids = [im.split_id for im in imgs]
    for shape in ("range", "terms"):
        hits = {}
        for field in ("client_ip", "client_u64"):
            req = request(shape, field)
            plans = [service.compile_plan(im, req, DM) for im in imgs]
            times = []
            for step in range(a.warmup + a.steps):
                r = ctx.split_search(ids, plans)
                if step >= a.warmup:
                    times.append(r[0].gpu_time_us)
            hits[field] = (sum(x.num_hits for x in r), sorted(c[0] for c in r[0].cells))
            print(json.dumps({"workload": f"ip_{shape}_{field}", "splits": a.splits, "docs_per_split": a.docs,
                              "device_us_p50": float(np.percentile(times, 50)), "device_us_p99": float(np.percentile(times, 99)),
                              "calls": a.steps, "num_hits": hits[field][0], "kernel_mask": r[0].kernel_mask,
                              "gpu": gpu[0] if gpu else "unknown", "build_s": round(build_s, 1)}), flush=True)
        # the twins compute the same thing: the same hit counts, and the same bucket counts
        assert hits["client_ip"][0] == hits["client_u64"][0], hits
        assert hits["client_ip"][1] == hits["client_u64"][1]
    ctx.close()


if __name__ == "__main__":
    main()
