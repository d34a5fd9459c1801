"""The posting-width sweep on the CPU: the corpora of posting_corpora.py realise the block widths they claim, the
oracle decodes every term back to its arrays, and the oracle agrees with scoring_ref on every query shape that
test_gpu_posting_widths.py sends to the GPU, bit for bit and within the f64 bound."""
import numpy as np
import pytest

from oracle import oracle as O
import posting_corpora as PC
import scoring_ref as R


@pytest.fixture(scope="module")
def sweep():
    return PC.sweep_split()


@pytest.fixture(scope="module")
def large():
    return PC.large_split()


@pytest.fixture(scope="module")
def tiny():
    return PC.tiny_split()


def _realised(c):
    out = {}
    for (f, t) in c.postings:
        s = PC.skips(c.img, c.img.term_ord(f, t))
        out[(f, t)] = [(int(x["doc_bits"]), int(x["tf_bits"]), int(x["count"])) for x in s]
    return out


def test_corpora_realise_the_widths_they_claim(sweep, large, tiny):
    """Every block's (doc_bits, tf_bits, count) in the image equals the one it was generated for, and together they
    cover doc widths 0..24 and tf widths 1..32."""
    doc_w, tf_w = set(), set()
    for c in (sweep, large, tiny):
        got = _realised(c)
        assert got == c.intended, [k for k in got if got[k] != c.intended[k]][:5]
        for (f, t), blocks in got.items():
            if t.startswith("w"):
                doc_w.update(b[0] for b in blocks)
            if t.startswith("tf"):
                tf_w.update(b[1] for b in blocks)
    assert sorted(doc_w) == list(range(25))
    assert sorted(tf_w) == list(range(1, 33))
    # phrase pairs at every doc width 0..22, tf widths up to 10
    ph = _realised(sweep)
    assert {b[0] for (f, t), bl in ph.items() if f == "ph" for b in bl} == set(range(23))
    assert {b[1] for (f, t), bl in ph.items() if f == "ph" for b in bl} == set(range(1, 11))
    # the tails: 1, 5 and 127 postings at every doc width
    for c, ws in ((sweep, range(23)), (large, (23, 24))):
        for w in ws:
            counts = {b[2] for t in c.terms_of("body", f"w{w:02d}_") for b in c.intended[("body", t)]}
            assert counts == {1, 5, 127, 128}, (w, counts)


def test_the_wide_delta_visits_every_position(sweep, large):
    """The largest delta 2^w - 1 sits at each of the 128 positions of a full block at widths 0..22 (at the lane,
    word and half-warp edges at 23 and 24), and the tf maximum 2^t - 1 is in every tf-sweep block."""
    for c, ws, want in ((sweep, range(1, 23), set(range(128))), (large, (23, 24), set(PC.LARGE_POSITIONS))):
        for w in ws:
            seen = set()
            for t in c.terms_of("body", f"w{w:02d}_"):
                docs = c.postings[("body", t)][0].astype(np.int64)
                v = np.diff(np.concatenate([[-1], docs])) - 1
                for i in range(0, len(v) - 127, 128):
                    blk = v[i:i + 128]
                    assert blk.max() == (1 << w) - 1
                    seen.update(np.flatnonzero(blk == (1 << w) - 1).tolist())
            assert want <= seen, (w, sorted(want - seen)[:8])
    for tw in range(1, 33):
        tfs = sweep.postings[("body", f"tf{tw:02d}")][1]
        for i in range(0, len(tfs), 128):
            assert int(tfs[i:i + 128].max()) == (1 << tw) - 1
    edge = sweep.postings[("body", "tf05_edge")][1]
    assert {14, 15, 16, 17} <= set(edge[:128].tolist())


def test_oracle_decodes_every_term(sweep, large, tiny):
    for c in (sweep, large, tiny):
        for (f, t), (docs, tfs, _) in c.postings.items():
            d, tf = O.decode_postings(c.img, c.img.term_ord(f, t), len(docs) + 1)
            assert np.array_equal(d, docs) and np.array_equal(tf, tfs), (c.split_id, f, t)


def test_oracle_unions_against_the_reference(sweep, large, tiny):
    """The k_union and k_window shapes: pure ORs (K = 1, 100, 4096), the mixed-width pairs, boosts, _score
    ascending, a `must` clause, and doc-id order (unscored)."""
    groups = PC.union_groups(sweep)
    for gi, g in enumerate(groups + PC.mixed_groups() + [PC.boosted(groups[0]), PC.boosted(groups[-3])]):
        for K, sort, must in ((1, "score_desc", None), (100, "score_desc", None), (4096, "score_desc", None),
                              (100, "score_asc", None), (4096, "doc_desc", None)):
            R.check(O.split_search(sweep.img, R.plan(sweep, g, K, sort, must)), sweep, g, K, sort, must, ctx=f"group {gi} {sort} K={K}")
    dense = R.Clause("body", ["dense"])
    for gi, g in enumerate(groups[:3]):
        gm = g[:31] + [dense]
        R.check(O.split_search(sweep.img, R.plan(sweep, gm, 100, must=len(gm) - 1)), sweep, gm, 100, must=len(gm) - 1, ctx=f"must {gi}")
    for c in (large, tiny):
        for g in PC.union_groups(c):
            for K in (1, 100, 4096):
                R.check(O.split_search(c.img, R.plan(c, g, K)), c, g, K, ctx=f"{c.split_id} K={K}")


def test_oracle_single_terms_against_the_reference(sweep):
    """The k_driver shape: one term, scored, with and without a range filter."""
    for f, t in PC.driver_terms(sweep):
        cl = [R.Clause(f, [t])]
        for filt in (False, True):
            R.check(O.split_search(sweep.img, R.plan(sweep, cl, 100, must=0, filt=filt)), sweep, cl, 100, must=0, filt=filt, ctx=f"{f}:{t} filt={filt}")


def test_oracle_phrases_against_the_reference(sweep):
    from quickwit_b200 import plan as P
    for cl in PC.phrase_pairs(sweep):
        for sort in ("score_desc", "doc_desc"):
            R.check(O.split_search(sweep.img, R.plan(sweep, [cl], 4096, sort, must=0)), sweep, [cl], 4096, sort, must=0, ctx=f"{cl.terms} {sort}")
    want = R.phrase_prefix_docs(sweep, "ph", "pa05_000", "pb")
    # (the oracle has no phrase-prefix node: it runs the same match set as an OR of one phrase per expansion)
    node = P.phrase_prefix(sweep.img, "ph", ["pa05_000", "pb"], 50)
    r = O.split_search(sweep.img, P.make_plan(P.phrase_prefix_as_phrases(node), 4096, R.SORTS["doc_desc"]))
    assert len(want) > 0 and r.num_hits == len(want) and [h[0] for h in r.hits] == want[::-1].tolist()
