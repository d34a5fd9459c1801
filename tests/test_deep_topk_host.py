"""Deep top-K (max_hits + start_offset up to 20 000) without a GPU.

qw_cand_cap (quickwit_b200/csrc/device_types.h) is the one rule for a split's candidate capacity that the host layout,
the candidate emitters and the threshold check share; it is compiled from the header into a small shared library, so
the test reads exactly what the engine reads. The oracle's paging identity pins what a deep request must return: the
page [s, s + 100) of a request is the slice of the single K = 20 000 list, on a corpus whose sort values tie."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from quickwit_b200 import ffi, plan as P, splitgen as S
from oracle import oracle as O
from helpers import col_sort

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM = ('#include "device_types.h"\n'
        'extern "C" unsigned cand_cap(unsigned k) { return qw_cand_cap(k); }\n'
        'extern "C" unsigned max_hits() { return QW_MAX_HITS; }\n')


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("cand_cap")
    (d / "shim.cpp").write_text(SHIM)
    cxx = os.environ.get("CXX", "g++")
    subprocess.run([cxx, "-O2", "-Wall", "-Werror", "-std=c++17", "-fPIC", "-shared", "-I", os.path.join(ROOT, "quickwit_b200", "csrc"),
                    "-o", str(d / "shim.so"), str(d / "shim.cpp")], check=True)
    lib = C.CDLL(str(d / "shim.so"))
    lib.cand_cap.argtypes, lib.cand_cap.restype = [C.c_uint], C.c_uint
    lib.max_hits.restype = C.c_uint
    return lib


def test_cand_cap_keeps_the_shallow_capacity(shim):
    for k in (0, 1, 10, 1000, 4095, 4096):
        assert shim.cand_cap(k) == 8192


def test_cand_cap_above_4096(shim):
    assert shim.max_hits() == 20000
    for k in list(range(4097, 4097 + 2048)) + [8192, 10000, 10001, 19999, 20000]:
        cap = shim.cand_cap(k)
        assert cap >= 2 * k and cap % 1024 == 0 and cap - 2 * k < 1024, (k, cap)
    assert shim.cand_cap(20000) == 40960


N = 60_000


@pytest.fixture(scope="module")
def tie_split():
    """Column a takes 40 values over 60 000 docs (ties of ~1500 docs at every K); b breaks some of them."""
    d = np.arange(N, dtype=np.int64)
    b = S._Builder(N)
    body = b.add_field("body", ffi.FIELD_HAS_FREQS | ffi.FIELD_HAS_FIELDNORMS, ffi.TOK_DEFAULT, np.full(N, 1, np.uint8), N)
    b.add_term(body, b"x", np.flatnonzero(d % 7 != 3).astype(np.uint32), np.ones(int((d % 7 != 3).sum()), dtype=np.uint32))
    a = ((d * 2654435761) % 40).astype(np.uint64)
    bb = ((d * 40503) % 3).astype(np.uint64)
    b.add_column("a", ffi.COL_U64, ffi.CARD_FULL, a, None)
    b.add_column("b", ffi.COL_U64, ffi.CARD_FULL, bb, None)
    return b.finish("deep-host-ties"), a, bb


@pytest.mark.parametrize("order", [ffi.ORDER_DESC, ffi.ORDER_ASC])
def test_oracle_pages_are_slices_of_the_deep_list(tie_split, order):
    img, a, bb = tie_split
    sort = [col_sort(img, "a", order), col_sort(img, "b", ffi.ORDER_ASC)]
    root = P.bool_([P.term(img, "body", "x", occur=ffi.OCCUR_MUST)])
    full = O.split_search(img, P.make_plan(root, 20000, sort))
    assert len(full.hits) == 20000
    # the full list against a brute force: a in the request's direction, b ascending, doc id in a's direction
    d = np.arange(N, dtype=np.int64)
    m = d % 7 != 3
    ka = -a.astype(np.int64) if order == ffi.ORDER_DESC else a.astype(np.int64)
    kd = -d if order == ffi.ORDER_DESC else d
    want = d[m][np.lexsort((kd[m], bb[m].astype(np.int64), ka[m]))][:20000]
    assert [h[0] for h in full.hits] == want.tolist()
    for s in list(range(0, 20000, 1900)) + [4000, 4096, 8150, 10000, 19900]:
        page = O.split_search(img, P.make_plan(root, s + 100, sort))
        assert page.num_hits == full.num_hits
        assert page.hits[s:s + 100] == full.hits[s:s + 100], f"page at {s}"
