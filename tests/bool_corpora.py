"""Splits for the boolean-program limits (test_bool_limits_host.py, test_gpu_bool_limits.py), built posting by posting
and column by column with splitgen._Builder from numpy arrays that bool_ref reads back (never the image).

Fields:
  * body: freqs and fieldnorms (128 fieldnorm bytes per posting block);
  * title: freqs, fieldnorms and positions (phrases);
  * tag: no freqs, no fieldnorms (a block is a 16-byte header plus the doc deltas: enough blocks in one window to
    pass QW_MAX_WBLK before the stage area fills);
  * extra: freqs and fieldnorms, for a third scored field.
Terms of body: `dense` (90 % of the docs, more than 160 blocks in every 32768-doc window, tfs up to 40), `heavy`
and `heavy2` (80 %, tfs up to 1000: each over the stage area by itself at every window size), m00..m15 (1 in 8 each: a few of them fill
the stage area at every window size), e0..e4 (the first and last doc of every window of 2048 << j docs, and the last
doc of the split), s00..s29 (about 300 docs each, tfs up to 20, some on window edges), `hitf` (tfs 16..5000).
Title: tt00..tt11 (5 %), `tdense` (50 %), the phrase pair pa / pb. Tag: a0..a5 (half the docs each, in 128 blocks per
32768-doc window).
Columns: `u` (FULL u64), `i` (OPTIONAL i64), c00..c14 (FULL u64, small)."""
from __future__ import annotations

import numpy as np

from quickwit_b200 import ffi, splitgen as S
from column_corpora import Col
from posting_corpora import Field

FN = ffi.FIELD_HAS_FREQS | ffi.FIELD_HAS_FIELDNORMS
N_MAIN = 16 * 32768 + 4097        # 17 windows of 32768 docs (a sampled threshold at every window size); not % 32
N_SMALL = 3001
WINDOWS = (2048, 4096, 8192, 16384, 32768)
I64_LO, I64_HI = -(1 << 40), 1 << 40


class BoolSplit:
    """The arrays of one split (scoring_ref's corpus interface: n, fields, postings; column_ref's: num_docs, cols,
    ords) and its image."""

    def __init__(self, n: int, split_id: str):
        self.n = self.num_docs = n
        self.split_id = split_id
        self.fields = {}
        self.postings = {}     # (field, term) -> (docs uint32, tfs uint32 or None, positions uint32 or None)
        self.cols = {}
        self.img = None
        self.ords = {}

    def build(self):
        b = S._Builder(self.n)
        fid = {}
        for f in self.fields.values():
            fid[f.name] = b.add_field(f.name, f.flags, ffi.TOK_DEFAULT, f.ids, f.total_tokens)
        for (field, name) in sorted(self.postings, key=lambda k: (fid[k[0]], k[1])):
            docs, tfs, pos = self.postings[(field, name)]
            b.add_term(fid[field], name.encode(), docs, tfs, pos)
        for name, c in self.cols.items():
            b.add_column(name, c.ctype, c.card, c.vals, c.index())
        self.img = b.finish(self.split_id)
        self.ords = {name: self.img.column_ord(name) for name in self.cols}
        return self

    def terms_of(self, field, prefix=""):
        return [t for (f, t) in sorted(self.postings) if f == field and t.startswith(prefix)]


def _pick(rng, n, p):
    return np.nonzero(rng.random(n) < p)[0].astype(np.uint32)


def _positions(rng, tfs, shift=None):
    """Positions 6 j + r_j (j < tf, r_j < 6) of every posting, distinct and ascending; `shift`: the same draws + 1."""
    tfs = tfs.astype(np.int64)
    j = np.arange(int(tfs.sum())) - np.repeat(np.cumsum(tfs) - tfs, tfs)
    r = rng.integers(0, 6, j.size) if shift is None else shift
    return (6 * j + r).astype(np.uint32), r


def make(n: int, split_id: str, seed: int, drop=()) -> BoolSplit:
    rng = np.random.default_rng(seed)
    c = BoolSplit(n, split_id)
    d = np.arange(n, dtype=np.int64)
    c.fields["body"] = Field("body", FN, rng.integers(0, 256, n).astype(np.uint8), 100 * n)
    c.fields["title"] = Field("title", FN | ffi.FIELD_HAS_POSITIONS, rng.integers(0, 40, n).astype(np.uint8), 12 * n)
    c.fields["tag"] = Field("tag", 0, None, 3 * n)
    c.fields["extra"] = Field("extra", FN, rng.integers(0, 256, n).astype(np.uint8), 50 * n)

    def add(field, name, docs, tfs=None, pos=None):
        if name in drop or len(docs) == 0:
            return
        docs = np.unique(np.asarray(docs, dtype=np.int64))
        docs = docs[(docs >= 0) & (docs < n)].astype(np.uint32)
        if field == "tag":
            tfs = None
        elif tfs is None:
            tfs = np.ones(docs.size, dtype=np.uint32)
        c.postings[(field, name)] = (docs, None if tfs is None else np.asarray(tfs[:docs.size], dtype=np.uint32), pos)

    def tf(k, lo, hi):
        return rng.integers(lo, hi + 1, k).astype(np.uint32)

    x = _pick(rng, n, 0.9)
    add("body", "dense", x, tf(x.size, 1, 40))
    for name in ("heavy", "heavy2"):
        x = _pick(rng, n, 0.8)
        add("body", name, x, tf(x.size, 1, 1000))
    for k in range(16):
        x = _pick(rng, n, 1 / 8)
        add("body", f"m{k:02d}", x, tf(x.size, 1, 12))
    for j in range(5):
        w = 2048 << j
        ks = np.arange(1, (n - 1) // w + 1) * w
        e = np.concatenate([[0, n - 1], ks - 1, ks])
        add("body", f"e{j}", e, tf(e.size + 2, 1, 3))
    for k in range(30):
        x = np.unique(rng.integers(0, n, max(3, n // 1800)))
        if k % 3 == 0:
            x = np.union1d(x, [0, n - 1, 2047, 2048, 32767, 32768][: 2 + k % 5])
        add("body", f"s{k:02d}", x, tf(x.size, 1, 20))
    x = np.unique(rng.integers(0, n, max(3, n // 250)))
    add("body", "hitf", x, tf(x.size, 16, 5000))

    for k in range(12):
        x = _pick(rng, n, 0.05)
        t = tf(x.size, 1, 3)
        add("title", f"tt{k:02d}", x, t, _positions(rng, t)[0])
    x = _pick(rng, n, 0.5)
    t = tf(x.size, 1, 2)
    add("title", "tdense", x, t, _positions(rng, t)[0])
    # pa / pb on the same docs: pb follows pa (a phrase) on about half of them
    x = _pick(rng, n, 0.04)
    t = tf(x.size, 1, 3)
    pa, r = _positions(rng, t)
    follow = np.repeat(rng.random(x.size) < 0.5, t)
    pb, _ = _positions(rng, t, shift=np.where(follow, r + 1, (r + 3) % 6))
    add("title", "pa", x, t, pa)
    add("title", "pb", x, t, pb)

    # a0 / a1: the even / odd docs (1-bit deltas); a2..a5: half of every 32768-doc window in one run (0-bit deltas)
    for k in range(6):
        x = d[d % 2 == k] if k < 2 else d[(d - 4096 * (k - 2)) % 32768 < 16384]
        add("tag", f"a{k}", x)
    for k in range(2):
        x = _pick(rng, n, 0.01)
        add("extra", f"x{k}", x, tf(x.size, 1, 5))

    c.cols["u"] = Col(ffi.COL_U64, ffi.CARD_FULL, rng.integers(0, 1 << 40, n, dtype=np.uint64), n)
    present = np.nonzero(rng.random(n) < 0.6)[0]
    iv = rng.integers(I64_LO, I64_HI, present.size)
    c.cols["i"] = Col(ffi.COL_I64, ffi.CARD_OPTIONAL, [S.i64_to_u64(int(v)) for v in iv], n, docs=present)
    for k in range(15):
        c.cols[f"c{k:02d}"] = Col(ffi.COL_U64, ffi.CARD_FULL, ((d * (7 + 2 * k)) % 1000 + k).astype(np.uint64), n)
    return c.build()


def main_split() -> BoolSplit:
    return make(N_MAIN, "bl-main", 0xB001)


SMALL_DROPS = ("dense", "pa", "m03", "m07", "s04", "a5", "tt05")


def small_split() -> BoolSplit:
    """A second split for batches: a few terms of the main split are missing."""
    return make(N_SMALL, "bl-small", 0xB002, drop=SMALL_DROPS)


# ---- the window index of the image, for the staging decision of k_window's phase 2 -------------------------------
WINIDX = np.dtype([("start", "<u4"), ("end", "<u4"), ("first_block", "<u4"), ("end_block", "<u4")])


def win_ranges(sp: BoolSplit, field: str, t: str, W: int):
    """(len, nb) per W-doc window of one term, as phase 1 of k_window reads them from the QwWinIdx entries: the byte
    range and the block count of the index windows the evaluation window overlaps. Zeros for an absent term."""
    nw = (sp.n + W - 1) // W
    o = sp.img.term_ord(field, t)
    if o < 0:
        return np.zeros(nw, dtype=np.int64), np.zeros(nw, dtype=np.int64)
    h = sp.img.header()
    tm = sp.img.terms()[o]
    nidx = (sp.n + (1 << tm.win_shift) - 1) >> tm.win_shift
    off = h.data_off + tm.widx_off
    wi = np.frombuffer(sp.img.array[off: off + 16 * nidx].tobytes(), dtype=WINIDX)
    ws = np.arange(nw, dtype=np.int64) * W
    we = np.minimum(ws + W, sp.n)
    a, b = wi[ws >> tm.win_shift], wi[(we - 1) >> tm.win_shift]
    ln = np.where(b["end"] > a["start"], b["end"].astype(np.int64) - a["start"], 0)
    nb = np.where((ln > 0) & (b["end_block"] > a["first_block"]), b["end_block"].astype(np.int64) - a["first_block"], 0)
    return ln, nb
