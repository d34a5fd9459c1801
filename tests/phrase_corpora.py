"""Splits built from numpy arrays with explicit positions, for the phrase, phrase-prefix and term-set pre-passes
(test_phrase_prepass_host.py, test_gpu_phrase_prepass.py). Each corpus keeps the arrays it was built from
(posting_corpora.Corpus: docs, tfs, positions per term; fieldnorm ids and total_tokens per field): phrase_ref computes
every expected result from them, never from the image.

`main_split()`, N_MAIN docs (not a multiple of 32), plants:
  * body: m1, m2 (a tenth of the docs each), r (rare, mostly inside m1 & m2), ta / tb (equal doc_freq), one (df 1),
    d128 / d129 (exactly 128 / 129 postings) and t1 / t5 / t127 (a tail block of 1, 5, 127 postings), r50 (a rare
    driver over them), sp (every 331st doc) beside dn (every 3rd: one sp block's candidates span ~110 dn blocks) and
    ea (ends at N / 2: later sp blocks find `lo == nblk`), ed beside lk (ed on lk's block last_docs, the next blocks'
    first docs and the gap after a last_doc). Positions of these are drawn from a few slots, so that phrases over
    them in any order and at any offsets match somewhere. ra / rb: runs `ra` x L and alternations `ra rb` x L for L
    in 1..40. ca / cb (also in nofn, a positions field without fieldnorms): phrase counts COUNTS over many
    fieldnorm ids.
  * far: fa / fb at positions FAR (0, 2^24 +- 1, 2^31 +- 1, ...), matching and off by one.
  * dp: `deep` with more than 2^24 positions before its later blocks, `dq` beside it in both parts.
  * mv: two values per doc with the multi-valued gap of one position between them (va vb | vc vd).
  * seq: the sentence s00..s11 at a few starting positions, some with the token after s00..s(k-1) replaced by an
    expansion sx0000..sx1024, some `s00 s00 s01`; every sx term also occurs alone elsewhere.
  * tsf (no positions): term-set terms on bitmap words 31/32/63/64, runs of 128 consecutive docs aligned and not
    to 32, tails of 1/31/32/33/127, two terms on one word from different blocks, the last doc of the split.
`offset_split()`: the three docs "a b", "x a b", "b a". `many_terms_split()`: 65 537 terms of one field.
`small_split(seed)`: a few thousand docs with short, long and prefix phrases and term sets, for batches over splits."""
from __future__ import annotations

import numpy as np

from quickwit_b200 import ffi
from posting_corpora import Corpus, FN

POS = FN | ffi.FIELD_HAS_POSITIONS
N_MAIN = 300_001
COUNTS = tuple(range(1, 18)) + (255, 256, 1000, 1500)
FAR = (0, 1, (1 << 24) - 1, 1 << 24, (1 << 24) + 1, (1 << 31) - 1, 1 << 31, (1 << 31) + 1, (1 << 31) + (1 << 24) + 3)
DEEP_DOCS, DEEP_TF = 4096, 4100   # 4096 * 4100 positions > 2^24 before the later blocks of `deep`
RUNS = tuple(range(1, 41))
N_SX = 1025
SEQ = [f"s{i:02d}" for i in range(12)]
WINDOWS = (2048, 4096, 8192, 16384, 32768)


class Plant:
    """Positions per (field, term, doc), turned into a Corpus's arrays."""

    def __init__(self, c):
        self.c, self.pos = c, {}

    def add(self, field, term, doc, positions):
        self.pos.setdefault((field, term), {}).setdefault(int(doc), set()).update(int(p) for p in positions)

    def finish(self):
        for key, per in self.pos.items():
            docs = np.array(sorted(per), dtype=np.uint32)
            tfs = np.array([len(per[d]) for d in docs.tolist()], dtype=np.uint32)
            pos = np.array([p for d in docs.tolist() for p in sorted(per[d])], dtype=np.uint32)
            self.c.postings[key] = (docs, tfs, pos)


def _rand_pos(rng, slots, tfmax=3):
    return rng.choice(slots, int(rng.integers(1, tfmax + 1)), replace=False)


def _subset(rng, docs, k):
    return np.sort(rng.choice(docs, k, replace=False))


def main_split(split_id="pp-main"):
    rng = np.random.default_rng(0x9A5E)
    n = N_MAIN
    c = Corpus(n, split_id)
    d = np.arange(n, dtype=np.int64)
    c.field("body", POS, ((d * 7 + 3) % 256).astype(np.uint8), 12 * n)
    c.field("nofn", ffi.FIELD_HAS_FREQS | ffi.FIELD_HAS_POSITIONS, None, 5 * n)
    c.field("far", POS, ((d * 3 + 1) % 256).astype(np.uint8), 40 * n)
    c.field("dp", POS, (d % 256).astype(np.uint8), 30 * n)
    c.field("mv", POS, ((d * 5 + 2) % 256).astype(np.uint8), 4 * n)
    c.field("seq", POS, ((d * 11 + 5) % 256).astype(np.uint8), 20 * n)
    c.field("tsf", ffi.FIELD_HAS_FREQS, None, 3 * n)
    c.field("wedge", POS, ((d * 7 + 2) % 256).astype(np.uint8), 6 * n)   # even ids on multiples of 2048
    pl = Plant(c)
    slots = np.arange(7)

    def scatter(field, term, docs, tfmax=3):
        for x in docs.tolist():
            pl.add(field, term, x, _rand_pos(rng, slots, tfmax))

    # ---- driver and lookup shapes -------------------------------------------------------------------------------
    m1 = np.flatnonzero(rng.random(n) < 0.1)
    m2 = np.sort(np.union1d(rng.choice(m1, len(m1) // 2, replace=False), np.flatnonzero(rng.random(n) < 0.05)))
    scatter("body", "m1", m1)
    scatter("body", "m2", m2)
    both = np.intersect1d(m1, m2)
    scatter("body", "r", np.union1d(_subset(rng, both, 380), _subset(rng, d, 20)), 2)
    scatter("body", "ta", _subset(rng, m1, 2000))
    scatter("body", "tb", _subset(rng, m1, 2000))
    one = int(both[len(both) // 2])
    pl.add("body", "one", one, [2])
    pl.add("body", "m1", one, [3])
    base = _subset(rng, m1, 700)
    for name, k in (("d128", 128), ("d129", 129), ("t1", 129), ("t5", 133), ("t127", 255)):
        scatter("body", name, _subset(rng, base, k))
    scatter("body", "r50", _subset(rng, base, 50), 2)
    sp = d[7::331]
    dn = d[1::3]
    ea = d[: n // 2][::2]
    scatter("body", "sp", sp)
    scatter("body", "dn", dn, 2)
    scatter("body", "ea", ea, 2)
    lk = d[::5]
    scatter("body", "lk", lk, 2)
    for i in range(0, 120, 3):
        last, nxt = int(lk[128 * i + 127]), int(lk[128 * (i + 1)])
        for x in (last, nxt, last + 2):          # last + 2: in the gap, not a doc of lk
            pl.add("body", "ed", x, [0, 4])
            if x % 5 == 0:
                pl.add("body", "lk", x, [1, 5])
    # ---- repeated terms: `ra` x L and `ra rb` x L ---------------------------------------------------------------
    rdocs = _subset(rng, d, 2 * len(RUNS))
    for L, x, y in zip(RUNS, rdocs[::2].tolist(), rdocs[1::2].tolist()):
        pl.add("body", "ra", x, range(3, 3 + L))
        pl.add("body", "ra", y, range(0, 2 * L, 2))
        pl.add("body", "rb", y, range(1, 2 * L, 2))
    # ---- phrase counts over many fieldnorm ids, with and without fieldnorms -------------------------------------
    cdocs = _subset(rng, d, 12 * len(COUNTS)).reshape(len(COUNTS), 12)
    for cnt, row in zip(COUNTS, cdocs):
        for x in row.tolist():
            for field in ("body", "nofn"):
                pl.add(field, "ca", x, range(0, 2 * cnt, 2))
                pl.add(field, "cb", x, range(1, 2 * cnt, 2))
    # ---- far positions ------------------------------------------------------------------------------------------
    fdocs = _subset(rng, d, 3 * len(FAR))
    for i, p in enumerate(FAR):
        a, b, e = fdocs[3 * i: 3 * i + 3].tolist()
        pl.add("far", "fa", a, [p])
        pl.add("far", "fb", a, [p + 1])
        pl.add("far", "fa", b, [p, p + 3])
        pl.add("far", "fb", b, [p + 1, p + 4])
        pl.add("far", "fa", e, [p])
        pl.add("far", "fb", e, [p + 2])
    # ---- a position stream past 2^24 entries ------------------------------------------------------------------
    late = _subset(rng, d[n // 2:], 600)
    deep_docs = np.concatenate([d[:DEEP_DOCS], late]).astype(np.uint32)
    deep_tf = np.concatenate([np.full(DEEP_DOCS, DEEP_TF), rng.integers(1, 4, len(late))]).astype(np.uint32)
    deep_pos = np.concatenate([np.tile(np.arange(DEEP_TF), DEEP_DOCS)] + [np.sort(rng.choice(8, t, replace=False)) for t in deep_tf[DEEP_DOCS:]])
    c.postings[("dp", "deep")] = (deep_docs, deep_tf, deep_pos.astype(np.uint32))
    for x in range(10, 4000, 97):
        pl.add("dp", "dq", x, [4000, 17])
    scatter("dp", "dq", _subset(rng, late, 300))
    # ---- multi-valued gap: "va vb" and "vc vd", the second value two positions after the first's last ---------
    for x in _subset(rng, d, 40).tolist():
        for t, p in (("va", 0), ("vb", 1), ("vc", 3), ("vd", 4)):
            pl.add("mv", t, x, [p])
    # ---- sentences and phrase-prefix expansions ---------------------------------------------------------------
    sdocs = _subset(rng, d, 900)
    for j, x in enumerate(sdocs.tolist()):
        st = j % 4
        toks = list(SEQ)
        if j >= 300:                                   # the token after s00..s(k-1) replaced by an expansion
            k = 1 + j % 7
            toks[k] = f"sx{[0, 1, 1022, 1023, 1024, int(rng.integers(0, N_SX))][(j // 7) % 6]:04d}"
        if j % 50 == 49:                               # s00 s00 s01 ...
            toks[1] = "s00"
        for i, t in enumerate(toks):
            pl.add("seq", t, x, [st + i])
    for k in range(N_SX):
        pl.add("seq", f"sx{k:04d}", int(rng.integers(0, n)), [100])
    # ---- window edges: `we wf` matches on every multiple of 2048 (the first doc of a window at every window size)
    # and on the doc after it; the driver's blocks hold the docs just before those too, so they straddle the edges
    for k in range(0, n // 2048 + 1):
        for x in (k * 2048 - 3, k * 2048 - 1, k * 2048, k * 2048 + 1) + ((1000,) if k == 0 else ()):  # (block starts off edges)
            if 0 <= x < n:
                on = x % 2048 in (0, 1)
                pl.add("wedge", "we", x, [0, 5])
                pl.add("wedge", "wf", x, [1, 6] if on else [2])
                pl.add("wedge", "wg", x, _rand_pos(rng, slots))
    # ---- term-set shapes ------------------------------------------------------------------------------------------
    ts = {}
    ts["w31"] = [31 * 32 + 5, 31 * 32 + 31]
    ts["w32"] = [32 * 32, 32 * 32 + 7]
    ts["w63"] = [63 * 32 + 31]
    ts["w64"] = [64 * 32, 64 * 32 + 30]
    ts["run_u"] = list(range(5000 + 8, 5000 + 8 + 128))               # crosses a word at each round boundary
    ts["run_a"] = list(range(32 * 300, 32 * 300 + 128))               # each round ends on a word boundary
    ts["run_a3"] = list(range(32 * 400, 32 * 400 + 3 * 128 + 32))
    for tail in (1, 31, 32, 33, 127):
        ts[f"tl{tail:03d}"] = list(range(20_000 + 1000 * tail, 20_000 + 1000 * tail + 3 * (128 + tail), 3))
    ts["sw_a"] = list(range(39_000, 39_000 + 127 * 7, 7)) + [40_000, 40_002]
    ts["sw_b"] = [40_001, 40_003] + list(range(41_000, 41_000 + 127 * 5, 5))
    ts["tend"] = list(range(n - 45, n))
    for t, docs in ts.items():
        for x in docs:
            pl.add("tsf", t, x, [0])
    pl.finish()
    for key in [k for k in c.postings if k[0] == "tsf"]:
        docs, tfs, _ = c.postings[key]
        c.postings[key] = (docs, tfs, None)
    return c.build()


def offset_split(split_id="pp-offsets"):
    """The docs "a b", "x a b" and "b a"."""
    c = Corpus(3, split_id)
    c.field("body", POS, np.array([2, 3, 2], dtype=np.uint8), 7)
    pl = Plant(c)
    for doc, text in enumerate(("a b", "x a b", "b a")):
        for i, t in enumerate(text.split()):
            pl.add("body", t, doc, [i])
    pl.finish()
    return c.build()


N_MANY = 70_001
MANY_TERMS = 65_537


def many_terms_split(split_id="pp-many"):
    """65 537 terms k00000.. of field k (no positions), term j on docs j % N_MANY and (7919 j + 13) % N_MANY."""
    c = Corpus(N_MANY, split_id)
    c.field("k", ffi.FIELD_HAS_FREQS, None, 2 * N_MANY)
    for j in range(MANY_TERMS):
        docs = np.unique(np.array([j % N_MANY, (7919 * j + 13) % N_MANY], dtype=np.uint32))
        c.postings[("k", f"k{j:05d}")] = (docs, np.ones(len(docs), dtype=np.uint32), None)
    return c.build()


def small_split(seed, split_id=None):
    """A few thousand docs: random sentences over a 12-token vocabulary in `body` (short and long phrases, phrase
    prefixes over the ten `v*` tokens) and term-set terms in `tsf`."""
    rng = np.random.default_rng(seed)
    n = 3000 + 1000 * (seed % 5)
    c = Corpus(n, split_id or f"pp-small-{seed}")
    d = np.arange(n, dtype=np.int64)
    c.field("body", POS, ((d * 13 + seed) % 256).astype(np.uint8), 20 * n)
    c.field("tsf", ffi.FIELD_HAS_FREQS, None, n)
    vocab = ["a", "b"] + [f"v{i}" for i in range(10)]
    pl = Plant(c)
    for x in range(n):
        L = int(rng.integers(2, 30))
        toks = rng.choice(vocab, L, p=[0.3, 0.3] + [0.04] * 10) if x % 7 else ["a", "b"] * (L // 2 + 1)
        for i, t in enumerate(toks):
            pl.add("body", str(t), x, [i])
        for j in range(int(rng.integers(0, 3))):
            pl.add("tsf", f"q{int(rng.integers(0, 40)):02d}", x, [0])
    pl.finish()
    for key in [k for k in c.postings if k[0] == "tsf"]:
        docs, tfs, _ = c.postings[key]
        c.postings[key] = (docs, tfs, None)
    return c.build()


def block_bounds(c, field, term):
    """(first doc, last doc) of every 128-posting block of a term, from the arrays."""
    docs = c.postings[(field, term)][0].astype(np.int64)
    starts = np.arange(0, len(docs), 128)
    return docs[starts], docs[np.minimum(starts + 127, len(docs) - 1)]


# ---- the queries of the GPU module (shared with the host module, which runs them on the oracle) ----------------------
def _expansions(k):
    return [f"sx{i:04d}" for i in range(k)]


def offset_cases():
    """(offsets (a, b), oracle docs) over offset_split: alignment alone decides, whatever the smallest offset."""
    return (((0, 1), [0, 1]), ((1, 2), [0, 1]), ((5, 6), [0, 1]), ((2, 1), [2]), ((9, 8), [2]), ((0, 4), []))


def main_queries():
    """(label, phrase_ref.Query) over main_split: each pre-pass clause alone, at its offsets, and inside bools."""
    from phrase_ref import Phrase as Ph, Prefix as Px, TermSet as TS, Term as T, Query as Q, MUST, SHOULD, FILTER, MUST_NOT
    qs = []

    def add(label, *clauses, msm=None):
        qs.append((label, Q(list(clauses), msm=msm, bare=len(clauses) == 1)))

    # driver and lookup shapes
    for terms in (["r", "m1", "m2"], ["m1", "r", "m2"], ["m1", "m2", "r"], ["ta", "tb"], ["tb", "ta", "m1"], ["one", "m1"],
                  ["m1", "one"], ["r50", "d128"], ["d128", "r50"], ["r50", "d129"], ["r50", "t127", "t5"], ["t1", "m1"],
                  ["t5", "m1"], ["t127", "m1"], ["d129", "m2"], ["sp", "dn"], ["dn", "sp"], ["sp", "ea"], ["ea", "sp", "dn"],
                  ["ed", "lk"], ["lk", "ed"], ["m1", "m2"]):
        add(f"shape {terms}", Ph("body", terms))
    # repeated terms
    for terms in (["ra", "ra"], ["ra", "rb", "ra"], ["ra"] * 8, ["rb", "ra", "rb"], ["ra"] * 9, ["ra", "rb"] * 5):
        add(f"repeat {terms}", Ph("body", terms))
    add("repeat ra@0 ra@2", Ph("body", ["ra", "ra"], [0, 2]))
    add("repeat ra@0 rb@1 ra@4", Ph("body", ["ra", "rb", "ra"], [0, 1, 4]))
    # offsets: gapped, above 0, not ascending, a driver whose positions lie below its offset
    for terms, offs in ((["r", "m1", "m2"], (0, 2, 5)), (["m1", "m2"], (1, 2)), (["m1", "m2"], (5, 6)), (["m1", "m2"], (2, 1)),
                        (["r", "m1", "m2"], (3, 0, 1)), (["r", "m1"], (5, 6)), (["r50", "d128"], (9, 7)),
                        (["sp", "dn"], (1000, 1001)), (["ed", "lk"], (3, 4)), (["va", "vb"], (4, 5)), (["ra", "rb"], (1, 0))):
        field = "mv" if terms[0] == "va" else "body"
        add(f"offsets {terms} {offs}", Ph(field, terms, offs))
    long_ = SEQ[:9]
    for offs in (range(9), range(1, 10), range(5, 14), range(8, -1, -1)):
        add(f"long offsets {list(offs)[:2]}..", Ph("seq", long_, list(offs)))
    add("long reversed", Ph("seq", long_[::-1], list(range(8, -1, -1))))
    gapped = [SEQ[i] for i in (0, 2, 3, 5, 6, 7, 8, 9, 11)]
    add("long gapped", Ph("seq", gapped, [0, 2, 3, 5, 6, 7, 8, 9, 11]))
    add("long gapped +5", Ph("seq", gapped, [5, 7, 8, 10, 11, 12, 13, 14, 16]))
    perm = [3, 0, 7, 1, 8, 2, 6, 4, 5]
    add("long permuted", Ph("seq", [SEQ[i] for i in perm], [i + 2 for i in perm]))
    add("long 12", Ph("seq", SEQ))
    # counts and norms, positions
    for field in ("body", "nofn"):
        add(f"counts {field}", Ph(field, ["ca", "cb"]))
        add(f"counts {field} reversed", Ph(field, ["cb", "ca"]))
        add(f"counts {field} @3,4", Ph(field, ["ca", "cb"], [3, 4]))
    for offs in ((0, 1), (5, 6), (1, 0), (0, 3), (2, 0)):
        add(f"far {offs}", Ph("far", ["fa", "fb"], offs))
    for terms, offs in ((["dq", "deep"], (0, 1)), (["deep", "dq"], (0, 1)), (["dq", "deep"], (3, 4)), (["deep", "dq"], (1, 0))):
        add(f"deep {terms} {offs}", Ph("dp", terms, offs))
    for terms, offs in ((["va", "vb"], (0, 1)), (["vb", "vc"], (0, 1)), (["vb", "vc"], (0, 2)), (["vc", "vd"], (0, 1))):
        add(f"multi-valued {terms} {offs}", Ph("mv", terms, offs))
    # phrase prefixes: k = 1..7 exact terms, 1 / 2 / 1023 / 1024 expansions, an expansion equal to an exact term,
    # offsets as above
    for k in range(1, 8):
        for e in (1, 2, 1023, 1024):
            add(f"prefix k={k} e={e}", Px("seq", SEQ[:k], _expansions(e), occur=FILTER))
    add("prefix k=1 e=1024 last only", Px("seq", ["s00"], ["sx1023"], occur=FILTER))
    add("prefix s00 s00*", Px("seq", ["s00"], ["s00", "s01"], occur=FILTER))
    add("prefix s00 + sx1024 (outside the 1024)", Px("seq", ["s00"], ["sx1024"], occur=FILTER))
    for offs, eo in (((1, 2), 3), ((5, 6), 7), ((2, 1), 3), ((0, 2), 4), ((4, 3), 2)):
        add(f"prefix offsets {offs} {eo}", Px("seq", ["s00", "s01"], ["s02", "s03", "sx0000"], list(offs), eo, occur=FILTER))
    add("prefix offsets 3 exact", Px("seq", ["s02", "s00", "s01"], _expansions(1023) + ["s03"], [5, 3, 4], 6, occur=FILTER))
    # term sets
    tsf = ["w31", "w32", "w63", "w64", "run_u", "run_a", "run_a3", "tl001", "tl031", "tl032", "tl033", "tl127", "sw_a", "sw_b", "tend"]
    add("term set all", TS("tsf", tsf))
    for grp in (["w31", "w32", "w63", "w64"], ["run_u"], ["run_a", "run_a3"], ["tl001", "tl031", "tl032", "tl033", "tl127"],
                ["sw_a", "sw_b"], ["tend"], ["sw_b"]):
        add(f"term set {grp}", TS("tsf", grp))
    # inside bools: MUST, SHOULD with minimum_should_match, FILTER, MUST_NOT, beside terms and the other pre-passes
    add("bool must+should", Ph("body", ["sp", "dn"], occur=MUST), T("body", "m1", SHOULD))
    add("bool should msm", Ph("body", ["m1", "m2"], occur=SHOULD), Ph("body", ["r", "m1"], [5, 6], occur=SHOULD), T("body", "r", SHOULD), msm=2)
    add("bool filter", Ph("body", ["m1", "m2"], [1, 2], occur=FILTER), T("body", "dn", MUST))
    add("bool must_not", T("body", "m1", MUST), Ph("body", ["m1", "m2"], [2, 1], occur=MUST_NOT))
    add("bool long+prefix", Ph("seq", long_, list(range(1, 10)), occur=SHOULD), Px("seq", ["s00"], _expansions(2), occur=FILTER),
        T("seq", "s05", SHOULD))
    add("bool term sets", T("body", "lk", MUST), TS("tsf", ["run_u", "tend"], occur=MUST_NOT), Ph("body", ["lk", "ed"], occur=SHOULD))
    return qs


def edge_queries():
    """(label, phrase_ref.Query) of the window-edge phrase `we wf`: MUST, SHOULD (also with minimum_should_match 2)
    and FILTER, and beside nested scored bools, whose accumulators shrink the window (engine.cu choose_route: the
    more score sums and levels, the smaller), so that together the scored and unscored runs reach every window size
    2048..32768."""
    from phrase_ref import Phrase as Ph, Term as T, Bool as B, Query as Q, MUST, SHOULD, FILTER

    def nest(depth):
        kids = [T("wedge", "wg", MUST), T("wedge", "we", SHOULD)]
        return B(kids + ([nest(depth - 1)] if depth > 1 else []), MUST)

    ph = lambda occ: Ph("wedge", ["we", "wf"], occur=occ)
    qs = [("edge must", Q([ph(MUST)], bare=True)),
          ("edge must+should", Q([ph(MUST), T("wedge", "wg", SHOULD)])),
          ("edge should", Q([ph(SHOULD), T("wedge", "wg", SHOULD)])),
          ("edge should msm 2", Q([ph(SHOULD), T("wedge", "wg", SHOULD), T("wedge", "we", SHOULD)], msm=2)),
          ("edge filter", Q([ph(FILTER), T("wedge", "wg", MUST), T("wedge", "we", SHOULD)]))]
    for depth in (1, 2, 3):
        qs.append((f"edge must, {depth + 1} levels", Q([ph(MUST), T("wedge", "wg", SHOULD), nest(depth)])))
        qs.append((f"edge should, {depth + 1} levels", Q([ph(SHOULD), T("wedge", "wg", MUST), nest(depth)])))
    return qs


def sorts_for(q):
    """(sort, K) pairs of a query; K = 0 is count-only. `_score` desc only where no phrase prefix or term set is a
    positive clause: the GPU refuses them in a scoring clause, and the oracle runs them as bools of phrases or terms."""
    unscorable = any(cl.kind in ("prefix", "term_set") and cl.occur != ffi.OCCUR_MUST_NOT for cl in q.clauses)
    out = [] if unscorable else [("score_desc", 1), ("score_desc", 10), ("score_desc", 1000), ("score_desc", 4096)]
    return out + [("doc_asc", 10), ("doc_desc", 1000), ("doc_asc", 4096), ("doc_desc", 0)]
