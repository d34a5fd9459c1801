"""Long phrases (9 to 64 tokens) on the GPU: device time of a call and the long-phrase pre-pass's share of it.

Two corpora, each served as --splits splits:
  * msg: BASELINE config 5's positions field (`synth_split(..., msg_vocab=64)`: 4 to 8 tokens per doc, Zipf over
    w0..w63). No document holds more than 8 tokens, so no long phrase matches there; its long phrases are the
    vocabulary's head `w0 w1 w2 ...` (the most frequent terms), and their rows time candidates that die after a few
    terms. `w1 w2` is the short-phrase control: its path is the one phrases of up to 8 tokens always took.
  * templated: log lines of 64 tokens whose first 12 tokens are one message template, in --template-share of the
    documents, followed by 52 Zipf draws over v0..v63; the other documents hold 8 Zipf draws. Phrases of 9, 16, 32
    and 64 tokens are cut from the start of one templated document, so a 9-token phrase matches every templated
    document (many candidates survive every term), and each is timed again with its last token changed (every
    candidate dies at the last term the pre-pass takes).

For each query: device time p50 / p99 over --steps calls of qwgpu_split_search over every split (the call's CUDA
events), then, in a separate profiled pass, the share of the call's device time spent in k_phrase / k_phrase_long
(torch.profiler, CUDA activities). Prints the card's name and power limit first, then one JSON line per query. Nothing
is written to the tree.

    python tools/bench_phrase_long.py
    python tools/bench_phrase_long.py --splits 4 --docs 200000 --steps 5   # a quick run
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TEMPLATE = ("info org apache hadoop hdfs server datanode datanode packetresponder receiving block blk").split()


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # (the timings stand without it)
        return {"gpu": "unknown", "error": str(e)}


def templated_split(num_docs, share, seed, split_id):
    """The templated corpus as one split image, and the tokens of its first templated document."""
    from quickwit_b200 import ffi, splitgen as S
    rng = np.random.default_rng(seed)
    vocab = [f"v{k}" for k in range(64)]
    zipf = 1.0 / np.arange(1, 65)
    tmpl = rng.random(num_docs) < share
    lens = np.where(tmpl, 64, 8).astype(np.int64)
    starts = np.cumsum(lens) - lens
    doc = np.repeat(np.arange(num_docs, dtype=np.int64), lens)
    pos = np.arange(int(lens.sum()), dtype=np.int64) - np.repeat(starts, lens)
    term = len(TEMPLATE) + rng.choice(64, size=len(pos), p=zipf / zipf.sum())  # ids: template slots, then v0..v63
    head = np.repeat(tmpl, lens) & (pos < len(TEMPLATE))
    names = TEMPLATE + vocab
    slot_term = np.array([names.index(t) for t in TEMPLATE])  # (`datanode` twice: one term id)
    term[head] = slot_term[pos[head]]
    order = np.lexsort((pos, doc, term))
    doc, pos, term = doc[order], pos[order], term[order]
    b = S._Builder(num_docs)
    L = ffi.img_lib()
    ids = {n: L.qwgpu_fieldnorm_to_id(n) for n in (8, 64)}
    fn = np.where(tmpl, ids[64], ids[8]).astype(np.uint8)
    fid = b.add_field("msg", ffi.FIELD_HAS_FREQS | ffi.FIELD_HAS_FIELDNORMS | ffi.FIELD_HAS_POSITIONS, ffi.TOK_DEFAULT,
                      fn, int(lens.sum()))
    bounds = np.searchsorted(term, np.arange(len(names) + 1))
    for t in sorted(range(len(names)), key=lambda i: names[i].encode()):
        lo, hi = bounds[t], bounds[t + 1]
        if lo == hi:
            continue
        d = doc[lo:hi]
        u, cnt = np.unique(d, return_counts=True)
        b.add_term(fid, names[t].encode(), u.astype(np.uint32), cnt.astype(np.uint32), pos[lo:hi].astype(np.uint32))
    first_doc = int(np.argmax(tmpl))
    sel = np.flatnonzero(doc == first_doc)
    tokens = [names[t] for t in term[sel][np.argsort(pos[sel])]]
    return b.finish(split_id), tokens


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--splits", type=int, default=32)
    ap.add_argument("--docs", type=int, default=3_125_000, help="docs per msg split")
    ap.add_argument("--template-docs", type=int, default=500_000, help="docs of the templated split (served --splits times)")
    ap.add_argument("--template-share", type=float, default=0.6)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile-steps", type=int, default=5)
    ap.add_argument("--k", type=int, default=10)
    a = ap.parse_args()
    from quickwit_b200 import ffi, plan as P, splitgen as S
    from quickwit_b200.service import SearcherContext

    print(json.dumps({"card": card()}), flush=True)
    ctx = SearcherContext(0)
    t = time.time()
    msg = []
    for i in range(a.splits):
        img = S.synth_split(a.docs, i, [0.2, 0.05], split_id=f"c5long-{i:03d}", msg_vocab=64)
        ctx.register_split(img)
        msg.append(img)
    timg, doc_tokens = templated_split(a.template_docs, a.template_share, 7, "tmpl-000")
    tmpl = [timg] + [S.SplitImage(timg.array, f"tmpl-{i:03d}") for i in range(1, a.splits)]
    for img in tmpl:
        ctx.register_split(img)
    build_s = time.time() - t
    sort = [(ffi.SORT_SCORE, ffi.ORDER_DESC, ffi.ABSENT)]

    def timed(imgs, plans):
        ids = [im.split_id for im in imgs]
        times, r = [], None
        for step in range(a.warmup + a.steps):
            r = ctx.split_search(ids, plans)
            if step >= a.warmup:
                times.append(r[0].gpu_time_us)
        return {"p50_us": round(float(np.percentile(times, 50)), 1), "p99_us": round(float(np.percentile(times, 99)), 1),
                "num_hits": sum(x.num_hits for x in r), "kernel_mask": r[0].kernel_mask}

    def prepass_share(imgs, plans):
        import torch
        from torch.profiler import ProfilerActivity, profile
        ids = [im.split_id for im in imgs]
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.profile_steps):
                ctx.split_search(ids, plans)
            torch.cuda.synchronize()
        dev = lambda e: getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        total = pre = 0.0
        for e in prof.key_averages():
            total += dev(e)
            if "k_phrase" in e.key:
                pre += dev(e)
        if total <= 0:
            return {"prepass_share": None, "note": "no device activity recorded"}
        return {"prepass_share": round(pre / total, 3), "prepass_us_per_call": round(pre / a.profile_steps, 1)}

    queries = [("msg", "w1 w2", ["w1", "w2"])]
    for n in (9, 16, 32, 64):
        queries.append(("msg", f"head {n}", [f"w{i}" for i in range(n)]))
    for n in (9, 16, 32, 64):
        cut = doc_tokens[:n]
        queries.append(("templated", f"cut {n}", cut))
        queries.append(("templated", f"cut {n}, last changed", cut[:-1] + ["v0" if cut[-1] != "v0" else "v1"]))
    for corpus, name, tokens in queries:
        imgs = msg if corpus == "msg" else tmpl
        plans = [P.make_plan(P.phrase(im, "msg", tokens), a.k, sort) for im in imgs]
        row = {"corpus": corpus, "query": name, "tokens": len(tokens), "splits": a.splits, "k": a.k, "calls": a.steps,
               "build_s": round(build_s, 1)}
        row.update(timed(imgs, plans))
        row.update(prepass_share(imgs, plans))
        print(json.dumps(row), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
