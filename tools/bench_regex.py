"""Regex queries on the GPU (DESIGN.md §4.8): device time of a call whose plans hold a regex's term set
(QW_NODE_TERM_SET: the k_term_set pre-pass, then k_window), against the same expansions as an OR-of-terms filter where
that plan exists (at most 64 terms), with the hits of both checked equal.

Workloads (one call over every split, 10 hits by doc id):
  * the config-5 corpus (--splits x --docs synthetic log docs, text field `msg` over w0 .. w63): `w1.*` (11 terms),
    `w[0-9]` (10) and `w.*` (64), each against bool{filter: bool{should: [the terms]}};
  * a high-cardinality field `hc` (--hc-splits x --hc-docs docs, one token each, about 100 000 distinct tokens
    h00000 .. h99999 per split): `h00[0-9]{3}` (1 000 terms) and `h0[0-9]{4}` (10 000), term set only.

Reported per workload: the host expansion time per split (the dictionary walk, as the compiler runs it), the
k_term_set kernel time (torch.profiler, in a separate pass), and the whole call's device time p50 / p99 (CUDA events),
with the card name and power limit read in the same run. Nothing is written to the tree.

    python tools/bench_regex.py
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

from quickwit_b200 import ffi, plan as P, service, splitgen as S  # noqa: E402
from quickwit_b200.service import SearcherContext  # noqa: E402

DOC_DESC = [(ffi.SORT_DOCID, ffi.ORDER_DESC, ffi.ABSENT)]


def hc_split(split_ord, n, seed):
    """`hc`: one token per doc, uniform over h00000 .. h99999 (about 20 docs per token at 2 M docs)."""
    rng = np.random.default_rng(seed + split_ord)
    tok = rng.integers(0, 100_000, n)
    order = np.argsort(tok, kind="stable")
    vals, starts = np.unique(tok[order], return_index=True)
    b = S._Builder(n)
    f = b.add_field("hc", 0, ffi.TOK_RAW, None, n)
    bounds = list(starts) + [n]
    for k, v in enumerate(vals):
        b.add_term(f, f"h{v:05d}".encode(), np.sort(order[bounds[k]:bounds[k + 1]]), None)
    return b.finish(f"hc-{split_ord:03d}")


def expand(imgs, field, pattern):
    """Per split: the expansion's term ords, and the host time of the walk."""
    out, secs = [], []
    for im in imgs:
        t = time.perf_counter()
        ords, _ = service.regex_terms(im, field, pattern)
        secs.append(time.perf_counter() - t)
        out.append(ords)
    return out, secs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--splits", type=int, default=32)
    ap.add_argument("--docs", type=int, default=3_125_000)
    ap.add_argument("--hc-splits", type=int, default=8)
    ap.add_argument("--hc-docs", type=int, default=2_000_000)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    ctx = SearcherContext(0)
    msg = [S.synth_split(a.docs, i, [0.2, 0.05], split_id=f"c5-{i:03d}", msg_vocab=64) for i in range(a.splits)]
    hc = [hc_split(i, a.hc_docs, 0x5EED) for i in range(a.hc_splits)]
    for im in msg + hc:
        ctx.register_split(im)
    hc_terms = [len(service.regex_terms(im, "hc", "h.*")[0]) for im in hc]

    workloads = []  # (name, imgs, term-set plans, OR-of-terms plans or None, host seconds per split, expansions)
    for field, imgs, pattern, with_or in (("msg", msg, "w1.*", True), ("msg", msg, "w[0-9]", True), ("msg", msg, "w.*", True),
                                          ("hc", hc, "h00[0-9]{3}", False), ("hc", hc, "h0[0-9]{4}", False)):
        ords, secs = expand(imgs, field, pattern)
        sets = [P.make_plan(P.term_set(im, field, o, ffi.OCCUR_MUST), 10, DOC_DESC) for im, o in zip(imgs, ords)]
        ors = None
        if with_or:
            ors = [P.make_plan(P.bool_([P.bool_([P.Node(ffi.NODE_TERM, ffi.OCCUR_SHOULD, term_ord=t) for t in o], occur=ffi.OCCUR_FILTER)]),
                               10, DOC_DESC) for o in ords]
        workloads.append((f"{field}:/{pattern}/", imgs, sets, ors, secs, [len(o) for o in ords]))

    times = {w[0]: {"set": [], "or": []} for w in workloads}
    for step in range(a.warmup + a.steps):
        for name, imgs, sets, ors, _s, _e in workloads:  # alternated: drift on the shared machine hits both plans alike
            ids = [im.split_id for im in imgs]
            r = ctx.split_search(ids, sets)
            if step >= a.warmup:
                times[name]["set"].append(r[0].gpu_time_us)
            if ors is not None:
                o = ctx.split_search(ids, ors)
                if step >= a.warmup:
                    times[name]["or"].append(o[0].gpu_time_us)
                if step == 0:
                    assert [(x.num_hits, x.hits) for x in r] == [(x.num_hits, x.hits) for x in o], name
            if step == 0:
                assert all(x.kernel_mask & ffi.KERNEL_TERM_SET for x in r), name

    # k_term_set alone, in a profiled pass of its own
    kernel_us = {}
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
        for name, imgs, sets, _o, _s, _e in workloads:
            ids = [im.split_id for im in imgs]
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    ctx.split_search(ids, sets)
            ev = [e for e in prof.events() if "k_term_set" in e.name]
            kernel_us[name] = sum(e.device_time for e in ev) / max(len(ev), 1) if ev else None
    except Exception as e:  # the profiler is optional: the call times above stand without it
        print(json.dumps({"profiler": f"unavailable: {e}"}), flush=True)

    for name, imgs, _sets, ors, secs, exps in workloads:
        t = times[name]
        row = {"workload": name, "splits": len(imgs), "docs_per_split": imgs[0].num_docs,
               "expansions_split0": exps[0], "host_expand_ms_per_split_p50": round(float(np.median(secs)) * 1e3, 3),
               "k_term_set_us": kernel_us.get(name), "device_us_p50": float(np.percentile(t["set"], 50)),
               "device_us_p99": float(np.percentile(t["set"], 99)), "calls": a.steps,
               "gpu": gpu[0] if gpu else "unknown"}
        if ors is not None:
            row.update({"or_of_terms_device_us_p50": float(np.percentile(t["or"], 50)),
                        "or_of_terms_device_us_p99": float(np.percentile(t["or"], 99)), "same_hits": True})
        if name.startswith("hc"):
            row["distinct_tokens_split0"] = hc_terms[0]
        print(json.dumps(row), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
