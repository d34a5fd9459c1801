"""qw_plan_score_hits (include/qwgpu_format.h): the plans whose hits the device returns as (doc id, score) pairs.
Only `_score` descending with no second key (or `_doc`, which extracts None), no search_after and QW_PLAN_FULL_HITS
clear; every other plan keeps full QwHit records. The predicate is compiled from the header into a small shared
library here, so the test reads exactly what the engine reads."""
import ctypes as C
import os
import subprocess

import pytest

from quickwit_b200 import ffi, plan as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM = '#include "qwgpu_format.h"\nint score_hits(const void* plan) { return qw_plan_score_hits((const QwPlanHeader*)plan); }\n'


@pytest.fixture(scope="module")
def score_hits(tmp_path_factory):
    d = tmp_path_factory.mktemp("score_hits")
    (d / "shim.c").write_text(SHIM)
    cc = os.environ.get("CC", "gcc")
    subprocess.run([cc, "-O2", "-Wall", "-Werror", "-fPIC", "-shared", "-I", os.path.join(ROOT, "include"),
                    "-o", str(d / "shim.so"), str(d / "shim.c")], check=True)
    fn = C.CDLL(str(d / "shim.so")).score_hits
    fn.argtypes, fn.restype = [C.c_char_p], C.c_int
    return lambda plan: fn(plan)


def _plan(sort, search_after=None, reserved=0):
    plan = P.make_plan(P.match_all(), 10, sort, search_after=search_after)
    if reserved:
        h = ffi.QwPlanHeader.from_buffer_copy(plan)
        h.reserved = reserved
        plan = bytes(h) + plan[C.sizeof(h):]
    return plan


SCORE_DESC = (ffi.SORT_SCORE, ffi.ORDER_DESC, ffi.ABSENT)
SCORE_ASC = (ffi.SORT_SCORE, ffi.ORDER_ASC, ffi.ABSENT)
DOC_DESC = (ffi.SORT_DOCID, ffi.ORDER_DESC, ffi.ABSENT)
DOC_ASC = (ffi.SORT_DOCID, ffi.ORDER_ASC, ffi.ABSENT)
COL = (ffi.SORT_COLUMN, ffi.ORDER_DESC, 0)
ABSENT_COL = (ffi.SORT_COLUMN, ffi.ORDER_ASC, ffi.ABSENT)


@pytest.mark.parametrize("sort, want", [
    ((SCORE_DESC,), 1),
    ((SCORE_DESC, DOC_DESC), 1),
    ((SCORE_DESC, DOC_ASC), 1),
    ((SCORE_ASC,), 0),
    ((SCORE_DESC, COL), 0),
    ((SCORE_DESC, SCORE_ASC), 0),
    ((SCORE_DESC, ABSENT_COL), 0),
    ((DOC_DESC,), 0),
    ((COL,), 0),
    ((COL, SCORE_DESC), 0),
])
def test_flag_follows_the_sort(score_hits, sort, want):
    assert score_hits(_plan(list(sort))) == want


def test_flag_is_clear_with_search_after_or_full_hits(score_hits):
    sa = ffi.QwSearchAfter()
    sa.present, sa.has_v1, sa.v1 = 1, 1, 0x8000000000000000
    assert score_hits(_plan([SCORE_DESC], search_after=sa)) == 0
    assert score_hits(_plan([SCORE_DESC], reserved=1)) == 0  # QW_PLAN_FULL_HITS
    assert score_hits(_plan([SCORE_DESC], reserved=2)) == 1
