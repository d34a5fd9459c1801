"""The cases of tests/test_gpu_select_edges.py checked without a GPU (tests/select_ref.py):
  * every case reaches what it was built for: branch, cut stop shift, candidates n, survivors m, shared bits `at`;
  * together they reach every target value of the module: each `at` of the sweep, each cut stop shift, m = 1..5, K
    above QW_SEL_MAX on the rank path, both branches, an all-zero key in a sorted-whole split;
  * the key restatement orders the matched docs as numpy's lexsort of the values does, and as the CPU oracle does.
The report (`pytest -s`) prints each case's restated path."""
import pytest

from oracle import oracle as O
import select_ref as R

CASES = [c for group in R.all_cases().values() for c in group]
ROUTES = ("window", "driver")


def _report(name, lab):
    print(f"[select-ref] {name:>24}: {lab}")


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_case_reaches_target(case):
    lab = case.label()
    _report(case.name, lab)
    t = case.target
    for key in ("branch", "stop", "n", "m", "common", "zero_key"):
        if t.get(key) is not None:
            assert getattr(lab, key) == t[key], f"{case.name}: {key} {getattr(lab, key)} != {t[key]} ({lab})"
    if "stop_below" in t:
        assert lab.stop is not None and lab.stop < t["stop_below"], f"{case.name}: {lab}"
    assert lab.n <= R.CAND_CAP


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_brute_force_against_lexsort_and_oracle(case):
    lay = case.layout()
    img = case.image(f"host-{case.name}")
    for name in case.vals:  # the key widths follow from the columns the image holds
        c, col = case.cols[name], img.columns()[img.column_ord(name)]
        assert (col.bits, col.min_value, col.gcd) == (c.bits, c.min, c.gcd), f"{case.name}: column {name}"
    if case.vals and case.num_docs > 1:
        assert lay.total_bits > 64, f"{case.name}: the first key word should not hold the whole key"
    want = lay.brute_docs(case.matched)
    assert want == lay.lexsort_docs(case.matched), f"{case.name}: key order differs from lexsort"
    for route in ROUTES:
        ref = O.split_search(img, case.plan(img, route))
        assert ref.num_hits == len(case.matched)
        assert [h[0] for h in ref.hits] == want[:case.K], f"{case.name} {route}: oracle differs from the brute force"


@pytest.mark.parametrize("name,sp,K,with_b", R.score_cases(), ids=[c[0] for c in R.score_cases()])
def test_score_case(name, sp, K, with_b):
    lay = sp.layout(with_b)
    docs = list(range(sp.n))
    want = lay.brute_docs(docs)
    assert want == lay.lexsort_docs(docs), f"{name}: key order differs from lexsort"
    img = sp.image(f"host-{name}")
    ref = O.split_search(img, sp.plan(img, K, with_b))
    assert [h[0] for h in ref.hits] == want[:K], f"{name}: oracle differs from the brute force"
    lab = R.restate(lay.keys(docs), K, lay.total_bits)
    _report(name, lab)
    assert lab.n <= R.CAND_CAP


def test_targets_covered():
    """Every value the GPU module is meant to reach is reached by at least one case."""
    labs = {c.name: c.label() for c in CASES}
    ats = {lab.at for lab in labs.values() if lab.branch == "rank"}
    want_at = set(R.AT_VALUE_TARGETS) | {p for p, _ in R.AT_DOC_TARGETS}
    assert want_at <= ats, sorted(want_at - ats)
    for p in (53, 117):  # the bucket bits cross each word boundary
        assert {p + i for i in range(11)} <= ats
    stops = {(lab.stop, lab.branch) for lab in labs.values()}
    for s in R.CUT_SHIFTS:
        assert (s, "rank") in stops and (s, "sort") in stops, s
    cut = {(lab.stop, lab.branch, lab.m) for c, lab in zip(CASES, labs.values()) if c.name.startswith("cut")}
    for s in R.CUT_SHIFTS:
        assert (s, "rank", 2048) in cut and (s, "sort", 2049 if s < 56 else 4096) in cut, s
    ms = {lab.m for lab in labs.values()}
    assert {1, 2, 3, 4, 5} <= ms
    rank_big_k = {c.K for c in CASES if c.K > R.SEL_MAX and labs[c.name].branch == "rank"}
    assert {2049, 3000, 4095, 4096} <= rank_big_k
    assert any(c.K == 2048 and labs[c.name].branch == "rank" and labs[c.name].stop is not None for c in CASES)
    # K > QW_SEL_MAX with more than K candidates: at least K > QW_SEL_MAX survive, so the split is sorted whole and the
    # cut's cap (K rounded up to 4096) never decides the result
    big = [labs[c.name] for c in CASES if c.K > R.SEL_MAX and labs[c.name].n > c.K]
    assert big and all(lab.branch == "sort" for lab in big)
    assert any(lab.zero_key and lab.branch == "sort" for lab in labs.values())
    pad = {lab.n for c, lab in zip(CASES, labs.values()) if c.name.startswith("pad")}
    assert pad == {2049, 3000, 4097, 8191}
    sc = [R.restate(sp.layout(wb).keys(range(sp.n)), K, sp.layout(wb).total_bits) for _, sp, K, wb in R.score_cases()]
    assert {lab.branch for lab in sc} == {"rank", "sort"}
    assert any(lab.m <= R.SEL_MAX for lab in sc) and any(lab.m > R.SEL_MAX for lab in sc)
