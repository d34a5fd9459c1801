"""The corpora of test_gpu_phrase_prepass.py realise the shapes they claim (read back from the image: skip entries,
position index), and the oracle agrees with phrase_ref's restatement on every plan of the GPU module, including every
offset case. No GPU needed."""
import numpy as np
import pytest

from oracle import oracle as O
from phrase_prefix_ref import rewrite_as_phrases
from regex_ref import rewrite_term_sets
import phrase_corpora as PC
import phrase_ref as Q
from posting_corpora import skips


@pytest.fixture(scope="module")
def main():
    return PC.main_split()


def _skips(c, field, term):
    return skips(c.img, c.img.term_ord(field, term))


def test_block_shapes(main):
    c = main
    for term, counts in (("one", [1]), ("d128", [128]), ("d129", [128, 1]), ("t1", [128, 1]), ("t5", [128, 5]),
                         ("t127", [128, 127])):
        assert _skips(c, "body", term)["count"].tolist() == counts, term
    assert len(c.postings[("body", "ta")][0]) == len(c.postings[("body", "tb")][0])
    for term in ("m1", "sp", "dn", "lk", "ed", "r"):
        sk = _skips(c, "body", term)
        first, last = PC.block_bounds(c, "body", term)
        assert sk["last_doc"].tolist() == last.tolist(), term
    # one sp block's candidates span dozens of dn blocks; ea's postings end before later sp blocks begin
    dn_last = _skips(c, "body", "dn")["last_doc"].astype(np.int64)
    first, last = PC.block_bounds(c, "body", "sp")
    spans = np.searchsorted(dn_last, last) - np.searchsorted(dn_last, first)
    assert spans.max() >= 100
    assert (first > int(c.postings[("body", "ea")][0][-1])).sum() >= 3
    # ed sits on lk's block last_docs, the next blocks' first docs and in the gaps after them
    lk_first, lk_last = PC.block_bounds(c, "body", "lk")
    ed = set(c.postings[("body", "ed")][0].tolist())
    lk = set(c.postings[("body", "lk")][0].tolist())
    assert len(ed & set(lk_last.tolist())) >= 30 and len(ed & set(lk_first.tolist())) >= 30 and len(ed - lk) >= 30
    # window edges: at every window size, every window's first doc (but doc 0) lies inside a block of the driver `we`
    # that starts before it, and `we wf` matches there
    f, l = PC.block_bounds(c, "wedge", "we")
    hits = set(Q.phrase_counts(c, "wedge", ["we", "wf"], [0, 1])[0].tolist())
    assert len(f) >= 4
    for w in PC.WINDOWS:
        for e in range(w, c.n, w):
            assert ((f < e) & (e <= l)).any() and e in hits, (w, e)


def test_positions_and_counts(main):
    c = main
    img = c.img
    # deep's position stream passes 2^24 entries before its later blocks, whose docs meet dq
    t = img.terms()[img.term_ord("dp", "deep")]
    h = img.header()
    pidx = np.frombuffer(img.array[h.data_off + t.pidx_off: h.data_off + t.pidx_off + 4 * (t.num_blocks + 1)].tobytes(), dtype="<u4")
    assert pidx[-1] == int(c.postings[("dp", "deep")][1].astype(np.int64).sum()) and pidx[-1] > (1 << 24)
    assert (pidx[:-1] > (1 << 24)).sum() >= 4
    late_hits = Q.phrase_counts(c, "dp", ["dq", "deep"], [0, 1])[0]
    assert (late_hits >= PC.DEEP_DOCS).sum() > 0 and (late_hits < PC.DEEP_DOCS).sum() > 0
    # phrase counts: every row of COUNTS over 12 fieldnorm ids, in both fields
    for field in ("body", "nofn"):
        d, n = Q.phrase_counts(c, field, ["ca", "cb"], [0, 1])
        assert sorted(set(n.tolist())) == sorted(PC.COUNTS)
        ids = c.fields["body"].ids
        for k in PC.COUNTS:
            assert len(set(ids[d[n == k]].tolist())) >= 10
    assert c.fields["nofn"].ids is None
    # far positions match at both edges of 2^24 and 2^31
    d, n = Q.phrase_counts(c, "far", ["fa", "fb"], [5, 6])
    fa = c.postings[("far", "fa")]
    assert len(d) == 2 * len(PC.FAR) and sorted(set(n.tolist())) == [1, 2]
    assert fa[2].max() >= (1 << 31) and fa[2].max() < (1 << 32) - (1 << 20)
    # term-set edges
    assert PC.N_MAIN % 32
    assert c.postings[("tsf", "tend")][0][-1] == PC.N_MAIN - 1
    for tail in (1, 31, 32, 33, 127):
        assert _skips(c, "tsf", f"tl{tail:03d}")["count"].tolist() == [128, tail]
    assert set(c.postings[("tsf", "sw_a")][0] // 32) & set(c.postings[("tsf", "sw_b")][0] // 32)


def test_restatement_of_offsets():
    """tantivy's rule on the three offset docs, restated and by the oracle."""
    c = PC.offset_split()
    for offs, want in PC.offset_cases():
        q = Q.Query([Q.Phrase("body", ["a", "b"], offs)], bare=True)
        assert Q.phrase_counts(c, "body", ["a", "b"], offs)[0].tolist() == want
        for sort in ("score_desc", "doc_asc"):
            Q.check(O.split_search(c.img, q.plan(c.img, 10, sort)), c, q, 10, sort, ctx=f"oracle offsets {offs}")


def test_oracle_agrees_with_restatement(main):
    """Every query of the GPU module, at every sort and K, on the oracle (nested bools included)."""
    for label, q in PC.main_queries() + PC.edge_queries():
        for sort, K in PC.sorts_for(q):
            pl = q.plan(main.img, K, sort)
            Q.check(O.split_search(main.img, rewrite_as_phrases(rewrite_term_sets(pl))), main, q, K, sort, ctx=f"{label} {sort} K={K}")
