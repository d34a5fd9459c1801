"""Term sets on the GPU (DESIGN.md §4.8): device time of calls whose query holds a set too large for the window
program's bool form, compiled from QueryAst as a leaf compiles it, so that the compiler's selection rule picks the form.

Workloads (one call over every split, 10 hits by doc id):
  * the config-5 corpus (--splits x --docs synthetic log docs):
      - `t1 AND tenant_id IN S`, |S| = 100 (the even ids 1000 .. 1198: half the corpus's tenants 1000 .. 1099, half
        outside the column's range; a COL_SET node, k_driver);
      - `t1 AND timestamp IN S`, |S| = 10 000 timestamps of the split (a COL_SET node, k_driver);
      - both sides of the selection: the wildcard `msg:w*` (all 64 `w` terms of the corpus: 64 TERM leaves, the bool
        form) and a term_set of those 64 terms plus `t0` (65 TERM leaves: a TERM_SET node);
  * an `ip` corpus (--ip-splits x --ip-docs docs, a fast `ip` column over 2^16 addresses): `client_ip IN` 10 000
    addresses (a COL_SET node, k_window's scan);
  * a high-cardinality text field (--hc-splits x --hc-docs docs, one token each over h00000 .. h99999): a wildcard
    `h00*` with 1 000 expansions (a TERM_SET node).

Reported per workload: the kernel route, the form the compiler chose, and the call's device time p50 / p99 (CUDA
events), with the card name and power limit read in the same run. Nothing is written to the tree.

    python tools/bench_term_sets.py
"""
import argparse
import ctypes as C
import ipaddress
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]

from quickwit_b200 import ffi, proto, service, splitgen as S  # noqa: E402
from quickwit_b200.service import SearcherContext  # noqa: E402

SYNTH_MAPPING = {"field_mappings": [{"name": "body", "type": "text"}, {"name": "msg", "type": "text"},
                                    {"name": "tenant_id", "type": "u64", "fast": True},
                                    {"name": "timestamp", "type": "datetime", "fast": True, "fast_precision": "nanoseconds"}]}
IP_MAPPING = {"field_mappings": [{"name": "client_ip", "type": "ip", "fast": True, "indexed": False}]}
HC_MAPPING = {"field_mappings": [{"name": "hc", "type": "text", "tokenizer": "raw"}]}
N_ADDR, IP_BASE = 1 << 16, int(ipaddress.IPv4Address("10.0.0.0"))


def ip_split(split_ord, n, seed):
    rng = np.random.default_rng(seed + split_ord)
    k = rng.integers(0, N_ADDR, n, dtype=np.uint64)
    present = np.unique(k)
    b = S._Builder(n)
    b.add_column("client_ip", ffi.COL_IP, ffi.CARD_FULL, np.searchsorted(present, k).astype(np.uint64), None,
                 [S.parse_ip(str(ipaddress.IPv4Address(IP_BASE + 251 * int(x)))) for x in present])
    return b.finish(f"ts-ip-{split_ord:03d}")


def hc_split(split_ord, n, seed):
    rng = np.random.default_rng(seed + split_ord)
    tok = rng.integers(0, 100_000, n)
    order = np.argsort(tok, kind="stable")
    vals, starts = np.unique(tok[order], return_index=True)
    b = S._Builder(n)
    f = b.add_field("hc", 0, ffi.TOK_RAW, None, n)
    bounds = list(starts) + [n]
    for k, v in enumerate(vals):
        b.add_term(f, f"h{v:05d}".encode(), np.sort(order[bounds[k]:bounds[k + 1]]), None)
    return b.finish(f"ts-hc-{split_ord:03d}")


def plan_nodes(plan):
    hs, ns = C.sizeof(ffi.QwPlanHeader), C.sizeof(ffi.QwPlanNode)
    h = ffi.QwPlanHeader.from_buffer_copy(plan[:hs])
    return [ffi.QwPlanNode.from_buffer_copy(plan[hs + i * ns: hs + (i + 1) * ns]) for i in range(h.num_nodes)]


def term_set(field, values):
    return {"type": "term_set", "terms_per_field": {field: list(values)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--splits", type=int, default=32)
    ap.add_argument("--docs", type=int, default=3_125_000)
    ap.add_argument("--ip-splits", type=int, default=8)
    ap.add_argument("--ip-docs", type=int, default=2_000_000)
    ap.add_argument("--hc-splits", type=int, default=8)
    ap.add_argument("--hc-docs", type=int, default=2_000_000)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    ctx = SearcherContext(0)
    synth = [S.synth_split(a.docs, i, [0.2, 0.05], split_id=f"ts-c5-{i:03d}", msg_vocab=64) for i in range(a.splits)]
    ips = [ip_split(i, a.ip_docs, 0x1B) for i in range(a.ip_splits)]
    hcs = [hc_split(i, a.hc_docs, 0x5EED) for i in range(a.hc_splits)]
    for im in synth + ips + hcs:
        ctx.register_split(im)

    rng = np.random.default_rng(3)
    ts_vals = [int(x) for x in rng.integers(1_700_000_000, 1_700_086_400, size=10_000)]  # seconds inside the splits' day
    w64 = [f"w{k}" for k in range(64)]  # (msg_vocab=64: w0 .. w63)

    def driver(field, values):
        return {"type": "bool", "must": [{"type": "term", "field": "body", "value": "t1"}], "filter": [term_set(field, values)]}

    workloads = [  # (name, imgs, mapping, ast)
        ("t1 AND tenant_id IN 100", synth, SYNTH_MAPPING, driver("tenant_id", range(1000, 1200, 2))),
        ("t1 AND timestamp IN 10000", synth, SYNTH_MAPPING, driver("timestamp", ts_vals)),
        ("msg:w* (64 expansions)", synth, SYNTH_MAPPING, {"type": "wildcard", "field": "msg", "value": "w*"}),
        ("msg IN 65 terms (set form)", synth, SYNTH_MAPPING, term_set("msg", w64 + ["t0"])),
        ("client_ip IN 10000", ips, IP_MAPPING,
         term_set("client_ip", [str(ipaddress.IPv4Address(IP_BASE + 251 * int(k))) for k in rng.choice(N_ADDR, 10_000, replace=False)])),
        ("hc:h00* (1000 expansions)", hcs, HC_MAPPING, {"type": "wildcard", "field": "hc", "value": "h00*"}),
    ]
    calls = []
    for name, imgs, mapping, ast in workloads:
        req = proto.enc_search_request(json.dumps(ast), max_hits=10, sort_fields=[("_doc", 1)])
        plans = [service.compile_plan(im, req, json.dumps(mapping)) for im in imgs]
        nodes = {n.kind for p in plans for n in plan_nodes(p)}
        form = "col_set" if ffi.NODE_COL_SET in nodes else "term_set" if ffi.NODE_TERM_SET in nodes else "bool"
        calls.append((name, [im.split_id for im in imgs], plans, form))

    times = {c[0]: [] for c in calls}
    masks = {}
    for step in range(a.warmup + a.steps):
        for name, ids, plans, _form in calls:  # alternated: drift on the shared machine hits every workload alike
            r = ctx.split_search(ids, plans)
            if step >= a.warmup:
                times[name].append(r[0].gpu_time_us)
            masks[name] = (r[0].kernel_mask, sum(x.num_hits for x in r))
    for name, ids, _plans, form in calls:
        t = times[name]
        mask, hits = masks[name]
        route = "k_driver" if mask & ffi.KERNEL_DRIVER else "k_window" if mask & ffi.KERNEL_WINDOW else hex(mask)
        print(json.dumps({"workload": name, "splits": len(ids), "form": form, "route": route,
                          "term_set_prepass": bool(mask & ffi.KERNEL_TERM_SET), "num_hits": hits,
                          "device_us_p50": float(np.percentile(t, 50)), "device_us_p99": float(np.percentile(t, 99)),
                          "calls": a.steps, "gpu": gpu[0] if gpu else "unknown"}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
