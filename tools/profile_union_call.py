#!/usr/bin/env python
"""Where the device time of one BM25-union search call goes: the bench's index (32 splits x 3.125 M docs, the
same splitgen seeds and plans as bench.py), the four C2 queries through seam C (`qwgpu_split_search`) under
torch.profiler with CUDA activities.

Writes under OUT:
  trace.pt.trace.json  the profiler's chrome trace;
  table.txt            per query: every memset / kernel / copy of the call in device order, its duration, the gap
                       before it, and for copies the bytes and achieved GB/s (median over the profiled repetitions);
                       the span from the call's first device operation after the plan upload to the end of its last
                       copy, which is what `gpu_time_us` (ev0 -> ev1) measures.
It also prints the card's name, power limit and SM clock. Tracing slows the host: take end-to-end numbers from
bench.py in a run of their own.

  python tools/profile_union_call.py [--reps 10] --out DIR
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card_info() -> str:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return f"nvidia-smi unavailable ({e})"


def device_ops(trace: dict):
    """GPU operations of the trace: (ts_us, dur_us, kind, name, bytes)."""
    ops = []
    for ev in trace.get("traceEvents", []):
        cat = ev.get("cat", "")
        if ev.get("ph") != "X" or cat not in ("kernel", "gpu_memcpy", "gpu_memset"):
            continue
        args = ev.get("args", {})
        ops.append((float(ev["ts"]), float(ev["dur"]), cat, ev.get("name", ""), int(args.get("bytes", 0) or 0)))
    ops.sort()
    return ops


def short(name: str) -> str:
    """`void qwk::k_union<1>(qwk::UParams)` -> `k_union<1>`; copies and memsets keep their names."""
    name = name.removeprefix("void ").replace("qwk::", "")
    head = name.split(">(")[0] + ">" if ">(" in name else name.split("(")[0]
    return head or name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10, help="profiled steps (each runs the four queries once)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)

    import torch
    from torch.profiler import ProfilerActivity, profile, record_function
    import bench
    from quickwit_b200.service import SearcherContext

    card = card_info()
    print(f"card: {card}", flush=True)
    torch.cuda.set_device(0)
    imgs = bench.build_splits(0, 32, 3_125_000, threads=min(os.cpu_count() or 1, 32))
    plans = bench.make_plans(imgs)
    ctx = SearcherContext(0)
    for img in imgs:
        ctx.register_split(img)
    ids = [im.split_id for im in imgs]
    searches = [bench.RawSearch(ctx, ids, plans[q]) for q in range(bench.Q_SETS)]
    for _ in range(a.warmup):
        for s in searches:
            s.run()
            s.free()
    torch.cuda.synchronize()

    calls = []  # (query, gpu_time_us, launches)
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for rep in range(a.reps):
            for q, s in enumerate(searches):
                with record_function(f"call q{q} r{rep}"):
                    r = s.run()
                s.free()
                calls.append((q, r["gpu_us"], r["launches"]))
    trace_path = os.path.join(a.out, "trace.pt.trace.json")
    prof.export_chrome_trace(trace_path)
    with open(trace_path) as f:
        trace = json.load(f)

    # the host range of every call: the call waits for its stream, so its device operations start and end inside it
    ranges = sorted((float(ev["ts"]), float(ev["ts"]) + float(ev["dur"]), ev["name"]) for ev in trace["traceEvents"]
                    if ev.get("ph") == "X" and str(ev.get("name", "")).startswith("call q") and ev.get("cat") == "user_annotation")
    ops = device_ops(trace)
    per_query = {}  # q -> list of per-call op lists
    for (t0, t1, name), (q, gpu_us, launches) in zip(ranges, calls):
        mine = [o for o in ops if t0 <= o[0] < t1]
        per_query.setdefault(q, []).append((mine, gpu_us, launches))

    lines = [f"card: {card}", f"reps: {a.reps} (median over them; times in us)", ""]
    for q in sorted(per_query):
        runs = per_query[q]
        shapes = {tuple((o[2], o[3]) for o in mine) for mine, _, _ in runs}
        lines.append(f"query {q}: gpu_time_us (ev0 -> ev1) median {statistics.median(g for _, g, _ in runs):.1f}, "
                     f"launches {runs[0][2]}, {len(shapes)} distinct op sequence(s)")
        mine0 = runs[0][0]
        n = min(len(m) for m, _, _ in runs)
        lines.append(f"  {'#':>2} {'kind':<10} {'name':<44} {'dur':>8} {'gap':>7} {'bytes':>9} {'GB/s':>7}")
        for i in range(n):
            kind, name, nbytes = mine0[i][2], mine0[i][3], mine0[i][4]
            dur = statistics.median(m[i][1] for m, _, _ in runs)
            gap = statistics.median(m[i][0] - (m[i - 1][0] + m[i - 1][1]) for m, _, _ in runs) if i else 0.0
            gbs = f"{nbytes / dur / 1e3:7.1f}" if nbytes and dur > 0 else ""
            lines.append(f"  {i:>2} {kind:<10} {short(name)[:44]:<44} {dur:8.1f} {gap:7.1f} {nbytes or '':>9} {gbs:>7}")
        # (the plan upload precedes ev0: the timed span starts at the op after the first host-to-device copy)
        first = 1 if n and mine0[0][2] == "gpu_memcpy" else 0
        span = statistics.median(m[n - 1][0] + m[n - 1][1] - m[first][0] for m, _, _ in runs)
        busy = statistics.median(sum(o[1] for o in m[first:n]) for m, _, _ in runs)
        lines.append(f"  span ops {first}..{n - 1}: {span:.1f} us, of which busy {busy:.1f} us, gaps {span - busy:.1f} us")
        lines.append("")
    text = "\n".join(lines)
    with open(os.path.join(a.out, "table.txt"), "w") as f:
        f.write(text + "\n")
    print(text)
    ctx.close()


if __name__ == "__main__":
    main()
