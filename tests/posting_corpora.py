"""Splits built posting by posting from numpy arrays, for the posting-decode and BM25 width sweep
(test_posting_widths_host.py, test_gpu_posting_widths.py).

Every posting block of a term is generated with the widths it is meant to have: its largest doc delta
(v = doc - previous doc - 1, BitPacker4x, qwgpu_format.h QwSkip) is exactly 2^w - 1 and its largest tf exactly
2^t - 1, every other value below. `intended[(field, term)]` lists (doc_bits, tf_bits, count) per block from those
parameters, not from the arrays, so that a builder that packed narrower than claimed is caught by comparing it with
the image's skip entries. A corpus keeps the arrays the split was built from (docs, tfs, positions per term; fieldnorm
ids and total_tokens per field): scoring_ref computes every expected result from them, never from the image.

  * `sweep_split()`: (1 << 22) + 4096 docs. Doc widths 0..22 with the wide delta at each of the 128 positions of a
    block (posting i sits in interleave lane i % 4, word i // 4; k_union's half-warp lane hl decodes 8 hl .. 8 hl + 7)
    plus tail blocks of 1, 5 and 127 postings; tf widths 1..32 (0xFFFFFFFF at 32), a block straddling the tf-factor
    table's 15 / 16 edge, a width-32 tf on a field with freqs and no fieldnorms; one dense term over every
    (fieldnorm id, tf 1..15) pair, also in a field whose f32 average fieldnorm exceeds 2^24; single-block terms in
    one k_union window whose widths put a narrow and a wide block in one warp step; phrase term pairs with identical
    doc lists at doc widths 0..22 and tf widths 1..10, with positions; a dense term for `must` clauses; column f.
  * `large_split()`: (1 << 24) + 256 docs, one text field, doc widths 23 and 24.
  * `tiny_split()`: one document holding two terms; `empty_split()`: no documents."""
from __future__ import annotations

import numpy as np

from quickwit_b200 import ffi, splitgen as S

N_SWEEP = (1 << 22) + 4096
N_LARGE = (1 << 24) + 256
UNION_W = 15360                       # k_union's window (engine.cu: 15360 * 2 / QU_MINB docs)
FN = ffi.FIELD_HAS_FREQS | ffi.FIELD_HAS_FIELDNORMS
TAILS = ((1, 0), (5, 3), (127, 126))  # (postings, position of the wide delta) of the partial blocks


class Field:
    def __init__(self, name, flags, ids, total_tokens):
        self.name, self.flags, self.ids, self.total_tokens = name, flags, ids, total_tokens


class Corpus:
    def __init__(self, n, split_id):
        self.n, self.split_id = n, split_id
        self.fields = {}          # name -> Field, in field-id order
        self.postings = {}        # (field, term) -> (docs uint32, tfs uint32, positions uint32 or None)
        self.intended = {}        # (field, term) -> [(doc_bits, tf_bits, count)] per block
        self.columns = {}
        self.img = None

    def field(self, name, flags, ids, total_tokens):
        self.fields[name] = Field(name, flags, ids, int(total_tokens))

    def term(self, field, name, blocks, positions=None):
        """blocks: [(deltas, tfs, doc_bits, tf_bits)], in doc order."""
        v = np.concatenate([b[0] for b in blocks]).astype(np.int64)
        docs = np.cumsum(v + 1) - 1
        assert docs[-1] < self.n, (name, int(docs[-1]))
        tfs = np.concatenate([b[1] for b in blocks]).astype(np.uint64)
        assert (tfs >= 1).all() and (tfs <= 0xFFFFFFFF).all()
        self.postings[(field, name)] = (docs.astype(np.uint32), tfs.astype(np.uint32), positions)
        self.intended[(field, name)] = [(b[2], b[3], len(b[0])) for b in blocks]

    def build(self):
        b = S._Builder(self.n)
        fid = {}
        for f in self.fields.values():
            fid[f.name] = b.add_field(f.name, f.flags, ffi.TOK_DEFAULT, f.ids, f.total_tokens)
        for (field, name) in sorted(self.postings):
            docs, tfs, pos = self.postings[(field, name)]
            b.add_term(fid[field], name.encode(), docs, tfs, pos)
        for name, vals in self.columns.items():
            b.add_column(name, ffi.COL_U64, ffi.CARD_FULL, vals, None)
        self.img = b.finish(self.split_id)
        return self

    def terms_of(self, field, prefix=""):
        return [t for (f, t) in sorted(self.postings) if f == field and t.startswith(prefix)]


def _block(rng, count, w, p, tw, q, small=4):
    """One block: deltas below min(2^w, small) but 2^w - 1 at position p; tfs in [1, 2^tw - 1] with 2^tw - 1 at q."""
    v = rng.integers(0, min(1 << w, small), count, dtype=np.int64)
    v[p] = (1 << w) - 1
    top = (1 << tw) - 1
    tf = rng.integers(1, top + 1, count, dtype=np.uint64) if top > 1 else np.ones(count, dtype=np.uint64)
    tf[q] = top
    return v, tf, w, tw


def _span(block):
    return int(block[0].sum()) + len(block[0])


def _width_terms(c, rng, field, prefix, w, positions, tails, tf_width, small=4):
    """Terms `prefix{w:02d}_{k:03d}` of doc width w: one full block per wide-delta position, packed greedily into
    as few terms as fit in the split, each tail block ending a term. Returns the term names."""
    positions = list(positions)
    marks = {len(positions) * (i + 1) // len(tails) - 1: t for i, t in enumerate(tails)}  # tails spread over the sequence
    units = []
    for i, p in enumerate(positions):
        units.append((128, p))
        if i in marks:
            units.append(marks[i])
    names, cur, used = [], [], 0

    def close():
        nonlocal cur, used
        if cur:
            name = f"{prefix}{w:02d}_{len(names):03d}"
            c.term(field, name, cur)
            names.append(name)
        cur, used = [], 0

    for j, (count, p) in enumerate(units):
        tw = tf_width(j)
        blk = _block(rng, count, w, p, tw, (p + 1 + j) % count, small)
        if used + _span(blk) > c.n:
            close()
        assert _span(blk) <= c.n
        cur.append(blk)
        used += _span(blk)
        if count < 128:
            close()
    close()
    return names


def _phrase_positions(rng, ta, tb):
    """Token positions of two terms in one document, drawn independently (the phrase count is what they give)."""
    L = 2 * max(ta, tb) + 2
    pa = np.sort(rng.choice(L, ta, replace=False)).astype(np.uint32)
    pb = np.sort(rng.choice(L + 1, tb, replace=False)).astype(np.uint32)
    return pa, pb


def sweep_split(split_id="pw-sweep"):
    rng = np.random.default_rng(0x5EED)
    n = N_SWEEP
    c = Corpus(n, split_id)
    d = np.arange(n, dtype=np.int64)
    # every fieldnorm id occurs; total_tokens is set, not summed, so that the averages are chosen: 200 tokens (body),
    # above 2^24 (big, where b * fieldnorm / avg rounds at high ids), 50 (ph); nofn has no fieldnorms (id 1 read)
    c.field("body", FN, (d % 256).astype(np.uint8), 200 * n)
    c.field("big", FN, ((d * 3 + 7) % 256).astype(np.uint8), n * ((1 << 25) + 12345))
    c.field("nofn", ffi.FIELD_HAS_FREQS, None, 7 * n)
    c.field("ph", FN | ffi.FIELD_HAS_POSITIONS, ((d * 5 + 1) % 256).astype(np.uint8), 50 * n)
    c.columns["f"] = (d % 10).astype(np.uint64)

    # doc-width sweep: tf widths 1..5 cycling over the blocks (the table path, and the divide path at 5)
    for w in range(23):
        _width_terms(c, rng, "body", "w", w, range(128), TAILS, lambda j: 1 + j % 5)

    # tf-width sweep: doc width 3, three full blocks and a tail of 5, the maximum tf at a different position each
    for tw in range(1, 33):
        c.term("body", f"tf{tw:02d}", [_block(rng, k, 3, (7 * i) % k, tw, (tw + 40 * i) % k) for i, k in enumerate((128, 128, 128, 5))])
    vs = rng.integers(0, 8, 128)
    vs[9] = 7
    c.term("body", "tf05_edge", [(vs, np.array([14, 15, 16, 17] * 32, dtype=np.uint64), 3, 5),
                                 (vs[::-1].copy(), np.array([16, 15] * 63 + [31, 1], dtype=np.uint64), 3, 5)])
    c.term("nofn", "tf32", [_block(rng, k, 4, i, 32, k - 1 - i) for i, k in enumerate((128, 128, 77))])
    c.term("nofn", "tf03", [_block(rng, k, 4, i + 5, 3, i) for i, k in enumerate((128, 128, 77))])

    # fieldnorm x tf table: docs 0..3839 = every (doc % 256 = fieldnorm id, tf = 1 + doc // 256) pair, in both
    # fieldnorm fields (big's ids are a permutation of the same 256 per 256 docs)
    fv = np.zeros(3840, dtype=np.int64)
    ftf = (1 + np.arange(3840) // 256).astype(np.uint64)
    for name in ("body", "big"):
        c.term(name, "fnsweep", [(fv[i:i + 128], ftf[i:i + 128], 0, int(ftf[i:i + 128].max()).bit_length())
                                 for i in range(0, 3840, 128)])
    # a dense term for `must` clauses (doc width 1: gaps of 1 and 2)
    dd = d[d % 3 != 0]
    dv = np.diff(np.concatenate([[-1], dd])) - 1
    dtf = (1 + dd % 13).astype(np.uint64)
    blocks = []
    for i in range(0, len(dd), 128):
        vv, tt = dv[i:i + 128], dtf[i:i + 128]
        blocks.append((vv, tt, int(vv.max()).bit_length(), int(tt.max()).bit_length()))
    c.term("body", "dense", blocks)

    # mixed-width warp steps: single-block terms whose postings sit in k_union window 1, except the wide delta
    def one(start, gap, wide_pos, wide, tfmax):
        v = np.full(128, gap - 1, dtype=np.int64)
        v[0] = start
        if wide:
            v[wide_pos] = (1 << wide) - 1
        tf = (1 + np.arange(128) % 15).astype(np.uint64)
        tf[64] = tfmax
        return v, tf, int(v.max()).bit_length(), int(tfmax).bit_length()

    c.term("body", "mx_n1", [one(UNION_W + 100, 3, 0, 0, 15)])          # 14 / 4 bits
    c.term("body", "mx_w1", [one(UNION_W + 50, 5, 127, 17, 15)])        # 17 / 4 bits: wide by its doc deltas
    c.term("body", "mx_n2", [one(UNION_W + 7, 4, 0, 0, 9)])             # 14 / 4 bits
    c.term("body", "mx_w2", [one(UNION_W + 11, 6, 0, 0, 1 << 20)])      # 14 / 21 bits: wide by its tfs
    c.term("body", "mx_n3", [one(UNION_W + 1, 2, 33, 16, 15)])          # 16 / 4 bits: the widest narrow block

    # phrase pairs pa / pb: identical doc lists at doc widths 0..22, tf widths 1..10, positions from a seeded draw
    for w in range(23):
        tmp = Corpus(n, "")
        names = _width_terms(tmp, rng, "ph", "x", w, (0, 45, 127), ((5, 3),), lambda j: 1 + (w + j) % 10)
        for k, nm in enumerate(names):
            docs, tfa, _ = tmp.postings[("ph", nm)]
            tfb = np.array([1 + (int(x) * 7 + w) % ((1 << (1 + (w + 3) % 10)) - 1) for x in tfa], dtype=np.uint32)
            pa, pb = zip(*[_phrase_positions(rng, int(x), int(y)) for x, y in zip(tfa, tfb)])
            blocks = tmp.intended[("ph", nm)]
            c.postings[("ph", f"pa{w:02d}_{k:03d}")] = (docs, tfa, np.concatenate(pa))
            c.postings[("ph", f"pb{w:02d}_{k:03d}")] = (docs, tfb, np.concatenate(pb))
            c.intended[("ph", f"pa{w:02d}_{k:03d}")] = blocks
            off = 0
            bb = []
            for (db, _tb, cnt) in blocks:
                bb.append((db, int(tfb[off:off + cnt].max()).bit_length(), cnt))
                off += cnt
            c.intended[("ph", f"pb{w:02d}_{k:03d}")] = bb
    return c.build()


LARGE_POSITIONS = (0, 1, 2, 3, 4, 7, 8, 15, 31, 32, 63, 64, 95, 96, 120, 126, 127)


def large_split(split_id="pw-large"):
    """Doc widths 23 and 24 (a 10 M-doc split reaches them): the wide delta at the lane, word and half-warp edges of
    a block, and the tails; the other deltas are 0 or 1 so that a width-24 block fits in 2^24 + 256 docs."""
    rng = np.random.default_rng(0x1A26E)
    n = N_LARGE
    c = Corpus(n, split_id)
    d = np.arange(n, dtype=np.int64)
    c.field("body", FN, ((d * 11) % 256).astype(np.uint8), 300 * n)
    for w in (23, 24):
        _width_terms(c, rng, "body", "w", w, LARGE_POSITIONS, TAILS, lambda j: 1 + j % 6, small=2)
    return c.build()


def tiny_split(split_id="pw-tiny"):
    c = Corpus(1, split_id)
    c.field("body", FN, np.array([37], dtype=np.uint8), 5)
    c.term("body", "w00_000", [(np.array([0]), np.array([3], dtype=np.uint64), 0, 2)])
    c.term("body", "w01_000", [(np.array([0]), np.array([70000], dtype=np.uint64), 0, 17)])
    return c.build()


def empty_split(split_id="pw-empty"):
    c = Corpus(0, split_id)
    c.field("body", FN, np.zeros(0, dtype=np.uint8), 0)
    return c.build()


SKIP = np.dtype([("last_doc", "<u4"), ("prev_last_doc", "<u4"), ("byte_off", "<u4"), ("doc_bits", "u1"),
                 ("tf_bits", "u1"), ("count", "<u2")])


def skips(img, term_ord):
    """The QwSkip entries of one term, read from the image."""
    h = img.header()
    t = img.terms()[term_ord]
    off = h.data_off + t.skip_off
    return np.frombuffer(img.array[off: off + 16 * t.num_blocks].tobytes(), dtype=SKIP)


# ---- the query shapes of the sweep (shared by the host and the GPU module) -------------------------------------------
def union_groups(c, field="body"):
    """Every doc- and tf-width term of `field` in clause groups of at most 32 (k_union's QU_MAX_TERMS), in name order
    (widths mixed within a group), then the fieldnorm x tf table over two fields and the field without fieldnorms."""
    from scoring_ref import Clause
    names = c.terms_of(field, "w") + c.terms_of(field, "tf")
    groups = [[Clause(field, [t]) for t in names[i:i + 32]] for i in range(0, len(names), 32)]
    if ("big", "fnsweep") in c.postings:
        groups.append([Clause("body", ["fnsweep"]), Clause("big", ["fnsweep"])])
        groups.append([Clause("nofn", ["tf32"]), Clause("body", ["tf32"]), Clause("nofn", ["tf03"]), Clause("body", ["tf05_edge"])])
    return groups


MIXED = (("mx_n1", "mx_w1"), ("mx_w1", "mx_n1"), ("mx_n2", "mx_w2"), ("mx_w2", "mx_n2"), ("mx_n1", "mx_w1", "mx_w2", "mx_n2"),
         ("mx_n3", "mx_w1"), ("mx_w1", "mx_n3"), ("mx_n3", "mx_w2"))


def mixed_groups():
    """Unions of single-block terms in k_union window 1: a narrow and a wide block in one warp step, both ways round."""
    from scoring_ref import Clause
    return [[Clause("body", [t]) for t in g] for g in MIXED]


def boosted(group, boosts=(0.5, 3.0, 1.7, 1.0, 0.25)):
    from scoring_ref import Clause
    return [Clause(cl.field, cl.terms, boosts[i % len(boosts)]) for i, cl in enumerate(group)]


def term_set_groups(c):
    """(field, terms) of the term sets over the sweep: one per doc width of `body` (its terms' blocks hold every
    wide-delta position and the tails), the tf-width sweep, and each other field's terms."""
    groups = [("body", c.terms_of("body", f"w{w:02d}_")) for w in range(23)]
    groups.append(("body", c.terms_of("body", "tf")))
    groups += [(f, c.terms_of(f)) for f in ("big", "nofn", "ph")]
    return groups


def driver_terms(c):
    return [(f, t) for (f, t) in sorted(c.postings) if f in ("body", "nofn", "big") and t != "dense"]


def phrase_pairs(c):
    from scoring_ref import Clause
    return [Clause("ph", [t, "pb" + t[2:]]) for t in c.terms_of("ph", "pa")]
