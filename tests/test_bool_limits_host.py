"""The cases of the boolean-program limits module (test_gpu_bool_limits.py), on the CPU:
  * the oracle agrees with bool_ref's restatement on every plan of the GPU module except the refusals (term sets
    reach the oracle as bools of SHOULD terms, regex_ref.rewrite_term_sets);
  * the restated shared-memory layout puts every call at the window size the GPU module asserts;
  * the split image realises the staging regimes the GPU module claims: phase 2 of k_window (kernels.cuh), restated
    from the image's QwWinIdx entries, stages a term when its window bytes fit the rest of the stage area, it has at
    most QW_BLK_TAB blocks in the window and the window's staged blocks stay within QW_MAX_WBLK; otherwise the term
    is decoded from global memory (direct mode). Terms are decided one after the other in program order."""
from __future__ import annotations

import time

import numpy as np
import pytest

from quickwit_b200 import ffi, plan as P
from regex_ref import oracle_search
import bool_corpora as BC
import bool_ref as B
import column_ref as CR

MUST, SHOULD, MUST_NOT, FILTER = B.MUST, B.SHOULD, B.MUST_NOT, B.FILTER
F32 = np.float32
SC_DESC = CR.Sort([(ffi.SORT_SCORE, ffi.ORDER_DESC, None)])
SC_ASC = CR.Sort([(ffi.SORT_SCORE, ffi.ORDER_ASC, None)])
BY_U = CR.col_sort("u", ffi.ORDER_ASC)
BY_I = CR.col_sort("i", ffi.ORDER_DESC, ("u", ffi.ORDER_ASC))
DOC_DESC = CR.SORT_DOC_DESC
U_MID = (1 << 38, 3 << 38)   # about half of column u

t_, ph, ts, rng, ex, al, bl = B.term, B.phrase, B.term_set, B.rng, B.exists, B.all_, B.bool_


def body(name, occur=MUST, **kw):
    return t_("body", name, occur, **kw)


def title(name, occur=MUST, **kw):
    return t_("title", name, occur, **kw)


def tag(name, occur=FILTER):
    return t_("tag", name, occur)


# ---- depth 4 -------------------------------------------------------------------------------------------------------
def deep_tree(scored: bool, msm0=None, msm3=None, level3_should=None):
    """Four bool levels; MUST, FILTER, SHOULD and MUST_NOT clauses at every level; scored term, phrase, range and
    match_all leaves at level 3; two sibling bools at levels 2 and 3; a nested MUST bool (level 1) whose MUST clause
    fails on docs its SHOULD clause matches. Unscored trees put term sets among the SHOULD clauses."""
    extra = [ts("title", ["tt06", "tt07"], SHOULD)] if not scored else []
    sh3 = level3_should if level3_should is not None else [
        ph("title", ["pa", "pb"], SHOULD, boost=1.5), rng("c02", 100, 700, SHOULD, boost=0.75),
        al(SHOULD, boost=0.125), body("m05", SHOULD)] + extra
    l3a = bl([body("m00"), rng("u", *U_MID, MUST, boost=0.5), title("tt00", FILTER), body("s00", MUST_NOT)] + sh3,
             msm=msm3, occur=SHOULD)
    l3b = bl([title("tt01", SHOULD), body("m01", SHOULD), ex("i", SHOULD, boost=2.0), body("e0", MUST_NOT),
              al(MUST, boost=0.25), rng("c03", 0, 899, FILTER)], occur=SHOULD)
    l2a = bl([body("m02"), l3a, l3b, title("tt02", SHOULD), body("s01", MUST_NOT), rng("c00", 50, 950, FILTER)],
             occur=SHOULD)
    l2b = bl([body("m03", SHOULD), body("m04", SHOULD), title("tdense", FILTER), tag("a1", MUST_NOT),
              bl([body("m06", SHOULD), title("tt03", SHOULD)], occur=FILTER), body("m07")], occur=MUST)
    # a MUST bool whose MUST clause (m08) misses docs that its SHOULD clause (m09) matches
    l1 = bl([l2a, l2b, body("m08"), body("m09", SHOULD), body("s02", MUST_NOT), ex("u", FILTER)], occur=MUST)
    l1s = bl([body("m10", SHOULD), bl([body("m11"), title("tt04", SHOULD)], occur=SHOULD), body("m12", MUST_NOT),
              rng("c01", 0, 600, FILTER), body("m13", SHOULD)], occur=SHOULD)
    return bl([l1, l1s, body("m14", SHOULD), tag("a0", FILTER), body("s03", MUST_NOT), body("dense")] + extra, msm=msm0)


def depth_calls(main):
    out = []
    sc = [(main, deep_tree(True), s, K, None) for s, K in ((SC_DESC, 1000), (SC_ASC, 100), (BY_U, 1000))]
    out.append(("depth 4 scored", 2048, sc))
    un = [(main, deep_tree(False), s, K, None) for s, K in ((BY_U, 1000), (DOC_DESC, 10), (BY_I, 4096))]
    out.append(("depth 4 unscored", 32768, un))
    return out


# ---- minimum_should_match ------------------------------------------------------------------------------------------
def msm_calls(main):
    out = []
    # level 0: SHOULD = term, duplicate term, phrase, range, nested bool (and a term set unscored)
    def l0(scored, msm):
        sh = [body("m00", SHOULD), body("m00", SHOULD), ph("title", ["pa", "pb"], SHOULD), rng("c04", 0, 299, SHOULD, boost=0.5),
              bl([body("m01"), title("tt00", SHOULD)], occur=SHOULD)]
        if not scored:
            sh.append(ts("title", ["tt01", "tt02", "tt03"], SHOULD))
        return bl([tag("a0")] + sh + [body("s00", MUST_NOT)], msm=msm), len(sh)
    for scored in (True, False):
        n = l0(scored, None)[1]
        items = [(main, l0(scored, m)[0], SC_DESC if scored else BY_U, 1000, None) for m in range(n + 2)]
        out.append((f"msm level 0 {'scored' if scored else 'unscored'}", 4096 if scored else 32768, items))
    # level 3 (the level-3 SHOULD clauses of deep_tree: phrase, range, match_all, term; plus a nested bool at level 4
    # is not allowed, so a duplicate term instead)
    for scored in (True, False):
        sh3 = [ph("title", ["pa", "pb"], SHOULD), rng("c02", 100, 700, SHOULD, boost=0.75), body("m05", SHOULD), body("m05", SHOULD),
               title("tt05", SHOULD)] + ([ts("title", ["tt06", "tt07"], SHOULD)] if not scored else [])
        items = [(main, deep_tree(scored, msm3=m, level3_should=sh3), SC_DESC if scored else BY_U, 100, None)
                 for m in range(len(sh3) + 2)]
        out.append((f"msm level 3 {'scored' if scored else 'unscored'}", 2048 if scored else 16384, items))
    # a term both MUST and MUST_NOT matches nothing
    both = bl([body("m02"), body("m02", MUST_NOT), body("m03", SHOULD)])
    out.append(("must and must_not", 8192, [(main, both, SC_DESC, 100, None), (main, both, BY_U, 100, None)]))
    return out


# ---- weights: IF_BITS_FROM_SCORE and around it ----------------------------------------------------------------------
TINY, HUGE = F32(1e-20), F32(1e30)
FMAX = np.finfo(np.float32).max


def boost_for(sp, name, target, side=0):
    """An f32 boost that gives body term `name` the f32 weight `target` (side 0), the largest weight below it (side
    -1) or the smallest weight at or above it (side 1), through the split's own idf."""
    df = sp.img.doc_freq(sp.img.term_ord("body", name))
    wt = lambda b: F32(P.bm25_weight(df, sp.n, float(b)))
    with np.errstate(over="ignore"):
        b = F32(F32(target) / wt(1.0))
    if side < 0:
        while wt(b) >= target:
            b = np.nextafter(b, F32(0))
        while np.isfinite(np.nextafter(b, F32(np.inf))) and wt(np.nextafter(b, F32(np.inf))) < target:
            b = np.nextafter(b, F32(np.inf))
    elif side > 0:
        while wt(b) < target:
            b = np.nextafter(b, F32(np.inf))
        while wt(np.nextafter(b, F32(0))) >= target:
            b = np.nextafter(b, F32(0))
    return float(b)


def weight_trees(sp):
    """(label, tree): should-term weights 0, just below and at or above 1e-20, just below and at or above 1e30,
    negative on a term and on a nested bool, two clauses whose f32 sum overflows to +inf (IF_BITS_FROM_SCORE is set
    for weights in [1e-20, 1e30) only)."""
    w = lambda name, target, side=0: body(name, SHOULD, boost=boost_for(sp, name, target, side))
    return [
        ("zero", bl([w("m00", 0.0), w("m01", 1.0)])),
        ("1e-20 edges", bl([w("m02", TINY, -1), w("m03", TINY, 1), title("tt00", SHOULD)])),
        ("only below 1e-20", bl([w("m05", TINY, -1), w("m06", TINY, -1)])),
        ("1e30 edges", bl([w("m07", HUGE, 1), w("m08", HUGE * F32(3)), w("m09", HUGE, -1)])),
        ("negative term", bl([w("m10", -2.5), w("m11", 1.0), body("s00", SHOULD)])),
        ("negative nested bool", bl([bl([w("m12", -3.0), title("tt01", SHOULD)], occur=SHOULD), w("m13", 0.5)])),
        ("overflow to +inf", bl([w("hitf", FMAX, -1), w("hitf", FMAX, -1), w("m14", 1.0)])),
        ("zero and negative with must", bl([body("m15"), w("m00", 0.0), w("m01", -1.0)])),
        # the best 1000 hold negative scores (threshold bucket 0); every score below -1 (no threshold)
        ("mostly negative", bl([w("m10", -2.5), body("s00", SHOULD)])),
        ("only negative", bl([w("s01", -40.0), w("s02", -40.0)])),
    ]


def weight_calls(main):
    items = [(main, q, s, 1000, None) for _, q in weight_trees(main) for s in (SC_DESC, SC_ASC, BY_U)]
    return [("weights", 4096, items)]


# ---- exactly at the limits, and one above -----------------------------------------------------------------------------
def limit_terms(main):
    """64 distinct terms of two scored fields: every body term but five, and 14 title terms."""
    bt = [t for t in main.terms_of("body") if t not in ("s25", "s26", "s27", "s28", "s29")]
    tt = main.terms_of("title")[:14]
    assert len(bt) == 50 and len(tt) == 14
    return [("body", t) for t in bt] + [("title", t) for t in tt]


def pure_or(terms, n=None):
    return bl([t_(f, x, SHOULD) for f, x in terms[:n]])


def limit_tree(terms, n_cols=16, n_instr=96, depth=4, extra_term=None, scored_field3=False):
    """A `depth`-level tree over `terms` (title terms at the deepest level), ranges over `n_cols` - 1 distinct columns
    (the sort column u is the last), padded with match_all clauses to `n_instr` instructions."""
    body_t = [t_(f, x, SHOULD) for f, x in terms if f == "body"]
    title_t = [t_(f, x, SHOULD) for f, x in terms if f == "title"]
    cols = (["i"] + [f"c{k:02d}" for k in range(15)])[:n_cols - 1]
    ranges = [rng(c, 0, 999, SHOULD, boost=0.5) if c != "i" else ex("i", SHOULD) for c in cols]
    leaf = title_t + ranges[:2]
    if extra_term is not None:
        leaf.append(extra_term)
    node = bl(leaf, occur=SHOULD)
    per = (len(body_t) + depth - 2) // max(depth - 1, 1)
    rest = body_t
    others = ranges[2:]
    for lv in range(depth - 2, -1, -1):
        chunk, rest = rest[:per], rest[per:]
        oc, others = others[:5], others[5:]
        node = bl(chunk + oc + [node] + (rest if lv == 0 else []) + (others if lv == 0 else []), occur=SHOULD if lv else MUST)
    if scored_field3:
        node.children.append(t_("extra", "x0", SHOULD))
    return node


def count_instr(q):
    return 1 if q.kind != "bool" else 2 + sum(count_instr(c) for c in q.children)


def pad_instr(q, n_instr):
    while count_instr(q) < n_instr:
        q.children.append(al(SHOULD, boost=0.0625))
    return q


def limit_calls(main):
    terms = limit_terms(main)
    out = []
    flat = pure_or(terms)
    assert count_instr(flat) == 66
    flat96 = pad_instr(bl(list(flat.children) + [rng(c, 0, 999, SHOULD, boost=0.5) if c != "i" else ex("i", SHOULD)
                                                  for c in ["i"] + [f"c{k:02d}" for k in range(14)]]), 96)
    tree = pad_instr(limit_tree(terms), 96)
    assert count_instr(flat96) == 96 and count_instr(tree) == 96
    out.append(("64 terms pure OR", 8192, [(main, flat, SC_DESC, K, None) for K in (10, 1000)] + [(main, flat, SC_ASC, 100, None)]))
    out.append(("96 instructions, 16 columns", 4096,
                [(main, q, s, 1000, None) for q in (flat96, tree) for s in (SC_DESC, BY_U)]))
    return out


def refusals(main):
    """(label, [items], message fragment): one over each limit."""
    terms = limit_terms(main)
    t65 = bl(list(pure_or(terms).children) + [tag("a0")])
    i97 = pad_instr(limit_tree(terms), 97)
    d5 = bl([bl([bl([bl([bl([body("m00"), body("m01", SHOULD)], occur=SHOULD), body("m02", SHOULD)], occur=SHOULD)],
                occur=SHOULD)], occur=SHOULD), body("m03")])
    f3 = bl([body("m00", SHOULD), title("tt00", SHOULD), t_("extra", "x0", SHOULD)])
    c17 = bl([rng(f"c{k:02d}", 0, 999, SHOULD) for k in range(15)] + [ex("i", SHOULD)])
    return [("65 terms", (main, t65, SC_DESC, 10, None), "more than 64 term clauses"),
            ("97 instructions", (main, i97, SC_DESC, 10, None), "97 > 96 instructions"),
            ("5 levels", (main, d5, BY_U, 10, None), "deeper than 4 levels"),
            ("3 scored fields", (main, f3, SC_DESC, 10, None), "more than 2 distinct text fields"),
            ("17 columns", (main, c17, BY_U, 10, None), "more than 16 columns")]


# ---- staging regimes ----------------------------------------------------------------------------------------------
REGIME_PLANS = {
    # every term direct: each alone is over the stage area (and, at 32768, over QW_BLK_TAB)
    "all direct": lambda: bl([body("dense"), body("heavy", SHOULD), body("heavy2", MUST_NOT)]),
    # every term staged: sparse terms
    "all staged": lambda: bl([body("e0"), body("s05", SHOULD), body("s06", SHOULD), body("e1", MUST_NOT)]),
    # the first m terms fill the stage area, the later ones go direct
    "overflow bytes": lambda: bl([body("m00"), tag("a0")] + [body(f"m{k:02d}", SHOULD) for k in range(1, 9)] +
                                 [body("m09", MUST_NOT), body("m10", MUST_NOT)]),
    # QW_MAX_WBLK: four 128-block tag terms fill the block table at 32768, the fifth goes direct with bytes to spare
    "overflow blocks": lambda: bl([tag("a0"), tag("a1", SHOULD), tag("a2", SHOULD), tag("a3", SHOULD),
                                   tag("a4", MUST_NOT), tag("a5", SHOULD)]),
    # one term over QW_BLK_TAB among staged ones
    "over blk_tab": lambda: bl([body("s07"), body("dense", SHOULD), body("m00", SHOULD), body("s08", MUST_NOT)]),
}
REGIMES_AT = {2048: ("all direct", "all staged", "overflow bytes"), 4096: ("all direct", "all staged", "overflow bytes"),
              8192: ("all direct", "all staged", "overflow bytes"), 16384: ("all direct", "all staged", "overflow bytes"),
              32768: ("all direct", "all staged", "overflow bytes", "overflow blocks", "over blk_tab")}
# plans that set a call's window size (the layout is the batch's largest)
SHAPERS = {
    32768: None,
    16384: lambda: bl([bl([body("m00", SHOULD), body("m01", SHOULD), body("m02", SHOULD)], msm=2, occur=SHOULD),
                       body("m03", SHOULD), body("m04", SHOULD)], msm=2),
    8192: lambda: bl([body("m00"), body("m01", SHOULD)]),
    4096: lambda: bl([body("m00"), bl([body("m01"), body("m02", SHOULD)], occur=SHOULD), body("m03", SHOULD)]),
    2048: lambda: bl([body("m00"), bl([body("m01"), bl([body("m02"), bl([body("m03"), body("m04", SHOULD)], occur=SHOULD)],
                                                     occur=SHOULD)], occur=SHOULD)]),
}


def regime_calls(main):
    out = []
    for W, names in REGIMES_AT.items():
        items = [(main, REGIME_PLANS[r](), BY_U, 1000, None) for r in names]
        if SHAPERS[W] is not None:
            items.append((main, SHAPERS[W](), BY_U if W == 16384 else SC_DESC, 100, None))
        out.append((f"staging W={W}", W, items))
    return out


def staging(sp, q, W):
    """Per window: [(term Q, staged, len, nb)] of phase 2 for the plan's term slots in program order."""
    slots = B.shape(sp, q, False, CR.Sort([])).slots
    per = [BC.win_ranges(sp, s.field, s.terms[0], W) for s in slots]
    cap = B.stage_bytes(W)
    out = []
    for w in range(len(per[0][0])):
        off = g = 0
        row = []
        for s, (ln, nb) in zip(slots, per):
            L, N = int(ln[w]), int(nb[w])
            ok = L > 0 and off + L <= cap and N <= B.BLK_TAB and g + N <= B.MAX_WBLK
            if ok:
                off += L
                g += N
            row.append((s, ok, L, N))
        out.append(row)
    return out


def regimes_of(sp, q, W):
    """The regimes phase 2 realises in some window of the split for plan q at window size W."""
    cap = B.stage_bytes(W)
    found = set()
    for row in staging(sp, q, W):
        live = [r for r in row if r[2] > 0]
        if len(live) < 2:
            continue
        if all(not ok for _, ok, _, _ in live):
            found.add("all direct")
        if all(ok for _, ok, _, _ in live):
            found.add("all staged")
        if any(N > B.BLK_TAB for _, _, _, N in live) and any(ok for _, ok, _, _ in live):
            found.add("over blk_tab")
        seen_staged = False
        for _s, ok, L, N in live:
            if ok:
                seen_staged = True
            elif seen_staged and L <= cap and N <= B.BLK_TAB:
                # direct only because the earlier terms used the room
                g = sum(r[3] for r in live if r[1])
                found.add("overflow blocks" if L <= cap - sum(r[2] for r in live if r[1]) and g + N > B.MAX_WBLK else "overflow bytes")
    return found


# ---- batches -----------------------------------------------------------------------------------------------------
def batch_call(main, small):
    l1 = bl([body("m00", SHOULD), title("tt00", SHOULD), rng("c05", 0, 499, SHOULD, boost=0.5)])
    l2 = bl([body("m01"), bl([body("m02", SHOULD), title("tt01", SHOULD)], occur=SHOULD), body("s00", MUST_NOT)])
    l3 = bl([bl([bl([body("m03", SHOULD), ph("title", ["pa", "pb"], SHOULD)], occur=MUST), body("m04", SHOULD)], occur=SHOULD),
             body("m05", SHOULD), ex("i", FILTER)])
    l4 = deep_tree(True)
    por = pure_or([("body", f"m{k:02d}") for k in range(6, 12)] + [("title", "tt02")])
    items = []
    k = 0
    Ks = (0, 1, 10, 1000, 4096)
    for sp in (main, small):
        for q in (l1, l2, l3, l4, por):
            items.append((sp, q, SC_DESC if k % 3 else SC_ASC, Ks[k % len(Ks)], None))
            k += 1
    items.append((main, l2, BY_I, 100, None))     # search_after from the restatement's 50th hit (set at run time)
    return [("batch", 2048, items)]


def with_search_after(items):
    """Sets the search_after of the last item from the restatement's 50th hit of its plan (K 100)."""
    sp, q, sort, K, _ = items[-1]
    mask, score = B.eval_split(sp, q)
    _, hits = CR.top_k(sp, mask, score, sort, 50)
    items[-1] = (sp, q, sort, K, CR.after(hits[-1]))
    return items


def all_calls(main, small):
    calls = depth_calls(main) + msm_calls(main) + weight_calls(main) + limit_calls(main) + regime_calls(main)
    b = batch_call(main, small)
    b[0] = (b[0][0], b[0][1], with_search_after(list(b[0][2])))
    return calls + b


# ---- the tests ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def splits():
    t = time.time()
    m, s = BC.main_split(), BC.small_split()
    print(f"[bool limits] splits built in {time.time() - t:.1f} s")
    return m, s


def test_corpus(splits):
    main, small = splits
    assert main.n % 32 and len(main.postings) >= 70
    assert len(main.fields) == 4 and len(main.cols) == 17
    docs = main.postings[("body", "dense")][0]
    assert np.count_nonzero(docs < 32768) >= 20481
    assert (main.postings[("body", "hitf")][1] > 16).all()
    for j in range(5):
        e = set(main.postings[("body", f"e{j}")][0].tolist())
        W = 2048 << j
        assert {W - 1, W, main.n - 1} <= e
    for t in BC.SMALL_DROPS:
        assert not any(k[1] == t for k in small.postings)
    # the threshold is sampled at 2048 and at 32768 docs per window: the stride over at least 16 windows
    for W in (2048, 32768):
        assert (main.n + W - 1) // W // 8 >= 2


def test_window_sizes(splits):
    main, small = splits
    reached = set()
    for label, W, items in all_calls(main, small):
        assert B.window_docs(items) == W, label
        reached.add(W)
    assert reached == set(BC.WINDOWS)


def test_limits_are_exact(splits):
    main, _ = splits
    terms = limit_terms(main)
    assert len({t for t in terms}) == 64
    tree = pad_instr(limit_tree(terms), 96)
    sh = B.shape(main, tree, True, BY_U)
    assert sh.n_instr == 96 and len(sh.slots) == 64 and len(sh.cols) == 16 and len(sh.fn_fields) == 2
    assert sh.levels == 0b1111
    assert B.shape(main, pure_or(terms), True, SC_DESC).fn_fields == ["body", "title"]


def test_weight_edges(splits):
    """The weight cases reach what they are named for: matches scored +inf, negative and 0."""
    main, _ = splits
    got = {}
    for label, q in weight_trees(main):
        m, s = B.eval_split(main, q)
        got[label] = s[m]
    assert np.isposinf(got["overflow to +inf"]).any()
    assert (got["negative term"] < 0).any() and (got["negative nested bool"] < 0).any()
    assert np.count_nonzero(got["mostly negative"] > 0) < 1000 <= got["mostly negative"].size
    assert (got["only negative"] < -1).any() and (got["only negative"] < 0).all() and got["only negative"].size < 1000
    assert (got["zero"] == 0).any() and (got["only below 1e-20"] > 0).all()


def test_staging_regimes(splits):
    """Every regime the GPU module claims occurs in some window, and each regime plan has required, SHOULD and
    MUST_NOT terms."""
    main, _ = splits
    for W, names in REGIMES_AT.items():
        for name in names:
            q = REGIME_PLANS[name]()
            occ = {c.occur for c in q.children}
            assert {SHOULD, MUST_NOT} <= occ and occ & {MUST, FILTER}, name
            assert name in regimes_of(main, q, W), (W, name, regimes_of(main, q, W))


def test_oracle_matches_restatement(splits):
    main, small = splits
    n = 0
    for label, _W, items in all_calls(main, small):
        for sp, q, sort, K, sa in items:
            pl = B.plan(sp, q, sort, K, sa)
            B.check(oracle_search(sp.img, pl), sp, q, sort, K, sa, ctx=f"{label} {sp.split_id} {q!r}")
            n += 1
    assert n > 50
