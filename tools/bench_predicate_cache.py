"""Paged search (search_after) through the predicate cache (DESIGN.md §4.9) on the config-5 corpus: 32 splits of
3.125 M docs per GPU, bench.build_splits' generator.

For each of four shapes, 20 pages of K = 100, each page after the last hit of the one before:
  * phrase  — msg:"w1 w2" within a time range, by timestamp desc;
  * regex   — msg:/w1.*/ AND body:t1, by timestamp desc;
  * and_not — config 5's body:t0 AND body:t1 AND NOT body:t4, by (tenant_id asc, timestamp desc);
  * driver  — body:t2 within a time range, by timestamp desc (k_driver's shape).
Seam C (qwgpu_split_search over every split, one batch per page, the plans compiled with the query in a `cache` node
as the leaf compiles a search_after request): device time per page (the call's CUDA events, gpu_time_us) with the
cache disabled, on a miss (the cache emptied before the page), and on a hit (the same page again), as p50 / p99 over
the pages; the miss's excess over the hit, as a share of the miss (the fill's share); bytes per entry. Seam A
(qwgpu_leaf_search with the protobuf request): host wall time per page, p50, disabled and warm.

The driver shape keeps k_driver under the route rule (no fill). To time the other side of the rule, the tool also
runs a plan it builds itself: bool{must: cache(the split's compiled query), must_not: match_none}. The must_not
clause changes no match but makes the plan ineligible for k_driver, so the cache serves it; both routes are confirmed
from kernel_mask. Card name and power limit are read in the same run. Prints one JSON object."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

T0 = 1_700_000_000
BUDGET = 4 << 30
HDR = None


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "not read"


def shapes(n_splits):
    span = 86_400 * n_splits
    term = lambda f, v: {"type": "term", "field": f, "value": v}
    phrase = {"type": "full_text", "field": "msg", "text": "w1 w2", "params": {"mode": {"type": "phrase"}}}
    rng = dict(start_timestamp=T0 + span // 4, end_timestamp=T0 + 3 * span // 4)
    by_ts = [("timestamp", 1)]
    return [
        ("phrase", phrase, dict(sort_fields=by_ts, **rng)),
        ("regex", {"type": "bool", "must": [{"type": "regex", "field": "msg", "regex": "w1.*"}, term("body", "t1")]}, dict(sort_fields=by_ts)),
        ("and_not", {"type": "bool", "must": [term("body", "t0"), term("body", "t1")], "must_not": [term("body", "t4")]},
         dict(sort_fields=[("tenant_id", 0), ("timestamp", 1)])),
        ("driver", {"type": "bool", "must": [term("body", "t2")]}, dict(sort_fields=by_ts, **rng)),
    ]


def pct(xs, q):
    return round(float(np.percentile(np.asarray(xs, dtype=np.float64), q)), 1) if xs else None


def guarded(plan: bytes) -> bytes:
    """bool{must: cache(the plan's query), must_not: match_none}: the same matches, not k_driver's shape."""
    from quickwit_b200 import ffi
    hsz, nsz = C.sizeof(ffi.QwPlanHeader), C.sizeof(ffi.QwPlanNode)
    h = ffi.QwPlanHeader.from_buffer_copy(plan[:hsz])
    nodes = [ffi.QwPlanNode.from_buffer_copy(plan[hsz + i * nsz:hsz + (i + 1) * nsz]) for i in range(h.num_nodes)]
    while nodes[0].kind == ffi.NODE_CACHE:  # (re-root on the query itself)
        nodes[0] = ffi.QwPlanNode.from_buffer_copy(bytes(nodes[nodes[0].first_child]))
    for n in nodes:
        if n.num_children:
            n.first_child += 3
    top = [ffi.QwPlanNode() for _ in range(3)]
    for n in top:
        n.boost, n.min_should_match, n.term_ord, n.column = 1.0, ffi.ABSENT, ffi.ABSENT, ffi.ABSENT
    top[0].kind, top[0].first_child, top[0].num_children = ffi.NODE_BOOL, 1, 2
    top[1].kind, top[1].occur, top[1].first_child, top[1].num_children = ffi.NODE_CACHE, ffi.OCCUR_MUST, 3, 1
    top[2].kind, top[2].occur = ffi.NODE_NONE, ffi.OCCUR_MUST_NOT
    nodes[0].occur = ffi.OCCUR_MUST
    tail = plan[hsz + h.num_nodes * nsz:]
    h.num_nodes = len(nodes) + 3
    return bytes(h) + b"".join(bytes(n) for n in top + nodes) + tail


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--splits", type=int, default=32)
    ap.add_argument("--docs-per-split", type=int, default=3_125_000)
    ap.add_argument("--pages", type=int, default=20)
    ap.add_argument("--k", type=int, default=100)
    a = ap.parse_args()
    from quickwit_b200 import ffi, proto, service
    from quickwit_b200.service import SearcherContext
    imgs = bench.build_splits(0, a.splits, a.docs_per_split, threads=min(os.cpu_count() or 1, 32), msg_vocab=bench.MSG_VOCAB)
    dm = json.dumps(bench.SYNTH_MAPPING)
    ctx = SearcherContext(0)
    for im in imgs:
        ctx.register_split(im)
    ids = [im.split_id for im in imgs]
    offsets = [proto.enc_split_offsets(im.split_id, im.num_docs) for im in imgs]
    out = {"card": card(), "splits": a.splits, "docs_per_split": a.docs_per_split, "pages": a.pages, "k": a.k, "shapes": {}}

    def leaf(ast, kw):
        lreq = proto.enc_leaf_search_request(proto.enc_search_request(json.dumps(ast), **kw), offsets, dm)
        t = time.perf_counter()
        resp = proto.dec_leaf_search_response(ctx.leaf_search(lreq))
        return resp, (time.perf_counter() - t) * 1e6

    def cold():
        ctx.set_predicate_cache_budget(0)
        ctx.set_predicate_cache_budget(BUDGET)

    for name, ast, kw in shapes(a.splits):
        kw = dict(kw, max_hits=a.k)
        ctx.set_predicate_cache_budget(0)
        # the pages' search_after values, from the leaf search with the cache disabled
        sas, sa = [], None
        for _ in range(a.pages):
            resp, _ = leaf(ast, dict(kw, search_after=sa) if sa else kw)
            if not resp["partial_hits"]:
                break
            sa = resp["partial_hits"][-1]
            sas.append(sa)
        # seam C: every page's plans (the cached query, as the leaf compiles a search_after request)
        cached = {"type": "cache", "inner": ast}
        pages = [[service.compile_plan(im, proto.enc_search_request(json.dumps(cached), **dict(kw, search_after=s)), dm) for im in imgs]
                 for s in sas]
        row = {"pages": len(pages)}
        variants = [("query", pages)]
        if name == "driver":
            variants.append(("guarded", [[guarded(p) for p in pl] for pl in pages]))
        for vname, vpages in variants:
            t_off, t_miss, t_hit, masks, same = [], [], [], set(), True
            for pl in vpages:
                ctx.set_predicate_cache_budget(0)
                ctx.split_search(ids, pl)  # (warm-up of the page's shape)
                r_off = ctx.split_search(ids, pl)
                cold()
                r_miss = ctx.split_search(ids, pl)
                r_hit = ctx.split_search(ids, pl)
                t_off.append(r_off[0].gpu_time_us)
                t_miss.append(r_miss[0].gpu_time_us)
                t_hit.append(r_hit[0].gpu_time_us)
                masks.add((r_off[0].kernel_mask, r_miss[0].kernel_mask, r_hit[0].kernel_mask))
                same &= all(x.num_hits == y.num_hits == z.num_hits and x.hits == y.hits == z.hits for x, y, z in zip(r_off, r_miss, r_hit))
            info = ctx.predicate_cache_info()
            row[vname] = {
                "seam_c_device_us": {"disabled": {"p50": pct(t_off, 50), "p99": pct(t_off, 99)},
                                     "miss": {"p50": pct(t_miss, 50), "p99": pct(t_miss, 99)},
                                     "hit": {"p50": pct(t_hit, 50), "p99": pct(t_hit, 99)}},
                "fill_share_of_miss": round(1 - pct(t_hit, 50) / pct(t_miss, 50), 3) if t_miss and pct(t_miss, 50) else None,
                "bytes_per_entry": info["used_bytes"] // info["entries"] if info["entries"] else None,
                "routes": sorted({"|".join(k for k, b in (("driver", ffi.KERNEL_DRIVER), ("window", ffi.KERNEL_WINDOW),
                                                          ("fill", ffi.KERNEL_PREDICATE_FILL)) if m & b) for ms in masks for m in ms}),
                "kernel_masks_off_miss_hit": sorted(f"{x:#x}/{y:#x}/{z:#x}" for x, y, z in masks),
                "results_identical": same,
            }
        # seam A: the same pages through qwgpu_leaf_search, disabled and with the cache warm
        a_off, a_on = [], []
        ctx.set_predicate_cache_budget(0)
        for s in sas:
            a_off.append(leaf(ast, dict(kw, search_after=s))[1])
        cold()
        for s in sas:
            leaf(ast, dict(kw, search_after=s))
            a_on.append(leaf(ast, dict(kw, search_after=s))[1])
        row["seam_a_wall_us_p50"] = {"disabled": pct(a_off, 50), "warm": pct(a_on, 50)}
        out["shapes"][name] = row
    ctx.set_predicate_cache_budget(0)
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
