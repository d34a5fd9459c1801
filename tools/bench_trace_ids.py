"""Jaeger trace search (find_trace_ids) on the GPU: device time of a Jaeger-shaped query over a synthetic span index.

Corpus: --splits splits of --docs spans; traces of 1..64 spans, adjacent in doc order, each with a fresh 16-byte trace id;
20 service names drawn Zipf(1.5) per trace; span timestamps over one hour at microsecond (--precision us) or second
(--precision s) precision — the second-precision corpus makes the N-th and (N+1)-th trace timestamps tie, which sends the
split through k_trace_replay. Query: service term AND start/end timestamp range AND duration range, num_traces N.

Prints one JSON line per N: device time p50 / p99 of the whole call (qwgpu_split_search over every split, CUDA events),
how many calls ran the replay, and the wall time of the Python restatement (tests/trace_ids_ref.py) on split 0.
Nothing is written to the tree.

    python tools/bench_trace_ids.py --precision us
    python tools/bench_trace_ids.py --precision s
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from quickwit_b200 import ffi, service, splitgen as S  # noqa: E402
from quickwit_b200.service import SearcherContext  # noqa: E402
from pipeline import search_request, term  # noqa: E402

T0 = 1_700_000_000
DM = {"field_mappings": [{"name": "service", "type": "text", "tokenizer": "raw"},
                         {"name": "trace_id", "type": "bytes", "fast": True},
                         {"name": "ts", "type": "datetime", "fast": True, "fast_precision": "microseconds"},
                         {"name": "dur", "type": "u64", "fast": True}], "timestamp_field": "ts"}


def build(split_ord, n, precision_ns, seed):
    rng = np.random.default_rng(seed + split_ord)
    runs = rng.integers(1, 65, n // 16 + 64)
    runs = runs[: int(np.searchsorted(np.cumsum(runs), n)) + 1]
    runs[-1] -= int(runs.sum()) - n
    nt = len(runs)
    ids = np.unique(rng.integers(0, 256, (nt, 16), dtype=np.uint8), axis=0)
    while len(ids) < nt:  # (collisions of random 128-bit ids do not happen in practice)
        ids = np.unique(np.vstack([ids, rng.integers(0, 256, (nt - len(ids), 16), dtype=np.uint8)]), axis=0)
    ords = rng.permutation(nt)
    doc_ord = np.repeat(ords, runs).astype(np.uint64)
    start = rng.integers(0, 3_600 * 10**9, nt)
    ts = (T0 * 10**9 + np.repeat(start, runs) + rng.integers(0, 10**9, n)).astype(np.int64)
    ts -= ts % precision_ns
    svc = np.repeat(np.minimum(rng.zipf(1.5, nt) - 1, 19), runs)
    b = S._Builder(n)
    fid = b.add_field("service", 0, ffi.TOK_RAW, None, n)
    for k in range(20):
        docs = np.nonzero(svc == k)[0].astype(np.uint32)
        if len(docs):
            b.add_term(fid, f"svc{k}".encode(), docs, None)
    b.add_column("trace_id", ffi.COL_BYTES, ffi.CARD_FULL, doc_ord, None, [bytes(r) for r in ids])
    b.add_column("ts", ffi.COL_DATETIME, ffi.CARD_FULL, (ts.view(np.uint64) ^ np.uint64(1 << 63)), None)
    dur = rng.integers(0, 10_000, n).astype(np.uint64)
    b.add_column("dur", ffi.COL_U64, ffi.CARD_FULL, dur, None)
    return b.finish(f"jaeger-{split_ord:03d}"), (svc, doc_ord, ts, dur)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--splits", type=int, default=32)
    ap.add_argument("--docs", type=int, default=3_125_000)
    ap.add_argument("--precision", choices=["us", "s"], default="us")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--num-traces", type=int, nargs="+", default=[20, 1000])
    a = ap.parse_args()
    prec = 1_000 if a.precision == "us" else 10**9
    ctx = SearcherContext(0)
    imgs, cols = [], []
    t = time.time()
    for i in range(a.splits):
        img, c = build(i, a.docs, prec, 0x7A11)
        ctx.register_split(img)
        imgs.append(img)
        if i == 0:
            cols.append(c)
    build_s = time.time() - t
    dm = json.dumps(DM)
    ast = {"type": "bool", "must": [term("service", "svc0"),
                                    {"type": "range", "field": "dur", "lower_bound": {"Included": 100}, "upper_bound": {"Included": 9_000}}]}
    lo, hi = T0 + 600, T0 + 3_000
    for n in a.num_traces:
        req = search_request(ast, start_timestamp=lo, end_timestamp=hi,
                             aggs={"num_traces": n, "trace_id_field_name": "trace_id", "span_timestamp_field_name": "ts"})
        plans = [service.compile_plan(im, req, dm) for im in imgs]
        ids = [im.split_id for im in imgs]
        times, replays = [], 0
        for step in range(a.warmup + a.steps):
            r = ctx.split_search(ids, plans)
            if step >= a.warmup:
                times.append(r[0].gpu_time_us)
                replays += bool(r[0].kernel_mask & ffi.KERNEL_TRACE_REPLAY)
        # the doc-by-doc restatement on split 0, same query
        import trace_ids_ref as R
        svc, doc_ord, ts, dur = cols[0]
        t = time.time()
        mask = (svc == 0) & (ts >= lo * 10**9) & (ts < hi * 10**9) & (dur >= 100) & (dur <= 9_000)
        R.select_trace_ids(zip(doc_ord[mask].tolist(), ts[mask].tolist()), n)
        oracle_s = time.time() - t
        print(json.dumps({"workload": "find_trace_ids", "precision": a.precision, "num_traces": n, "splits": a.splits,
                          "docs_per_split": a.docs, "device_us_p50": float(np.percentile(times, 50)),
                          "device_us_p99": float(np.percentile(times, 99)), "calls": a.steps, "calls_with_replay": replays,
                          "python_restatement_split0_s": round(oracle_s, 3), "build_s": round(build_s, 1)}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
