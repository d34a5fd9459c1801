"""BM25-union top-K calls large enough to give every block of the collect pass at least four windows sample their
threshold inside that pass (k_union<MODE_SAMPLE_COLLECT>): each block's first window is the sample, the blocks meet
at a grid barrier, and each picks the same threshold from the complete histogram. Such a call issues two kernel
launches (the collect pass and k_select) and reports sample_stride = windows // grid. Results must equal the oracle's
on that path, on the two-launch path a batch falls back to when one split holds no block's first window, and through
the exact repair when a tie overflows the candidate capacity. The eligibility rule and the per-split sample weights
(qw_fused_sample_plan, device_types.h) are pinned without a GPU."""
import ctypes as C
import os
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from quickwit_b200 import ffi, plan as P, splitgen as S
from oracle import oracle as O
from helpers import assert_same

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W = 15360            # docs per k_union window
BLOCKS_PER_SM = 2    # QU_MINB
N_SPLITS = 9
DOCS = 2_100_000     # 137 windows per split: 9 x 137 = 1233 >= 4 x 264 blocks on an H100 SXM
FRACS = [0.2, 0.1, 0.05, 0.02, 0.01]


def chunk_begin(total, b, grid):
    return total * b // grid


def windows(num_docs):
    return (num_docs + W - 1) // W


# ---- the rule, without a GPU ------------------------------------------------------------------------------------------
SHIM = ('#include "device_types.h"\n'
        'extern "C" int plan(const unsigned* fw, const unsigned* mh, unsigned n, unsigned grid, unsigned* stride) {\n'
        '  return qw_fused_sample_plan(fw, mh, n, grid, stride) ? 1 : 0;\n}\n')


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("fused_sample")
    (d / "shim.cpp").write_text(SHIM)
    cxx = os.environ.get("CXX", "g++")
    subprocess.run([cxx, "-O2", "-Wall", "-Werror", "-std=c++17", "-fPIC", "-shared", "-I", os.path.join(ROOT, "quickwit_b200", "csrc"),
                    "-o", str(d / "shim.so"), str(d / "shim.cpp")], check=True)
    lib = C.CDLL(str(d / "shim.so"))
    lib.plan.restype = C.c_int
    return lib


def _plan(shim, wins, grid, max_hits=None):
    n = len(wins)
    fw = np.concatenate([[0], np.cumsum(wins)]).astype(np.uint32)
    mh = np.array(max_hits if max_hits is not None else [10] * n, dtype=np.uint32)
    stride = np.zeros(n, dtype=np.uint32)
    ok = shim.plan(fw.ctypes.data_as(C.c_void_p), mh.ctypes.data_as(C.c_void_p), n, grid, stride.ctypes.data_as(C.c_void_p))
    return bool(ok), stride.tolist()


def _expected(wins, grid, max_hits=None):
    """The rule restated: samples of a split = blocks whose chunk begins in it."""
    fw = np.concatenate([[0], np.cumsum(wins)])
    total = int(fw[-1])
    if total < 4 * grid:
        return False, None
    begins = [chunk_begin(total, b, grid) for b in range(grid)]
    ok, strides = True, []
    for s, nw in enumerate(wins):
        samples = sum(1 for w in begins if fw[s] <= w < fw[s + 1])
        if nw and (max_hits is None or max_hits[s]) and not samples:
            ok = False
        strides.append(max(1, nw // samples) if samples else 1)
    return ok, strides if ok else None


def test_fused_sample_rule(shim):
    # the bench's batch: 32 splits x 204 windows over 132 SMs x 2 blocks -> 8 or 9 samples per split
    ok, st = _plan(shim, [204] * 32, 264)
    assert ok and (ok, st) == _expected([204] * 32, 264) and set(st) == {204 // 8, 204 // 9}
    # this file's batch
    ok, st = _plan(shim, [137] * 9, 264)
    assert ok and (ok, st) == _expected([137] * 9, 264)
    # fewer than four windows per block: the two-launch path
    assert _plan(shim, [131] * 8, 264)[0] is False and _expected([131] * 8, 264)[0] is False
    assert _plan(shim, [10], 0)[0] is False
    # a one-window split that no chunk begins in: not eligible, unless it asks for no hits
    wins = [137, 1] + [137] * 8
    assert chunk_begin(sum(wins), 29, 264) < 137 < chunk_begin(sum(wins), 30, 264)
    assert _plan(shim, wins, 264)[0] is False and _expected(wins, 264)[0] is False
    ok, st = _plan(shim, wins, 264, max_hits=[10, 0] + [10] * 8)
    assert ok and st == _expected(wins, 264, [10, 0] + [10] * 8)[1] and st[1] == 1
    # (with 8 equal splits over 264 = 8 x 33 blocks every split starts a chunk: a one-window split there is sampled)
    assert _plan(shim, [137, 1] + [137] * 7, 264)[0] is True
    # empty splits (no windows) do not count, wherever they sit
    wins = [0, 137, 0, 0] + [137] * 7 + [0]
    ok, st = _plan(shim, wins, 264)
    assert ok and (ok, st) == _expected(wins, 264) and st[0] == st[2] == st[3] == st[-1] == 1
    # uneven splits: each split's weight is its own windows over its own samples, rounded down
    wins = [1000, 57, 300, 40]
    ok, st = _plan(shim, wins, 64)
    assert ok and (ok, st) == _expected(wins, 64) and st[0] > st[1] >= 1
    # (a 9-window split between chunk starts 21 windows apart holds none)
    assert _plan(shim, [1000, 57, 300, 9], 64)[0] is _expected([1000, 57, 300, 9], 64)[0] is False


# ---- on the GPU -------------------------------------------------------------------------------------------------------
def _grid():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * BLOCKS_PER_SM


@pytest.fixture(scope="module")
def corpus(gpu_ctx):
    imgs = [S.synth_split(DOCS, i, FRACS, split_id=f"fused-{i}") for i in range(N_SPLITS)]
    for im in imgs:
        gpu_ctx.register_split(im)
    yield imgs
    for im in imgs:
        gpu_ctx.unregister_split(im.split_id)


def _or_plan(img, K, terms=("t0", "t1", "t2", "t3")):
    root = P.bool_([P.term(img, "body", t, occur=ffi.OCCUR_SHOULD) for t in terms])
    return P.make_plan(root, K, [(ffi.SORT_SCORE, ffi.ORDER_DESC, ffi.ABSENT)])


def _path(r):
    return (f"kernel_mask={r.kernel_mask:#x} sample_stride={r.sample_stride} launches={r.num_kernel_launches} "
            f"exact_fallbacks={r.exact_fallbacks} radix_passes={r.radix_passes}")


def _check(res, imgs, plans, tag):
    for i, (r, im, pl) in enumerate(zip(res, imgs, plans)):
        assert r.kernel_mask & ffi.KERNEL_UNION and not r.kernel_mask & ffi.KERNEL_WINDOW or r.exact_fallbacks, f"{tag}: {_path(r)}"
        assert_same(r, O.split_search(im, pl), ctx=f"{tag} split {i}")


@pytest.mark.gpu
@pytest.mark.parametrize("K", [10, 1000, 4096])
def test_fused_sample_matches_oracle(gpu_ctx, corpus, K):
    grid = _grid()
    total = N_SPLITS * windows(DOCS)
    assert total >= 4 * grid, "the batch must qualify for the fused sample on this card"
    plans = [_or_plan(im, K) for im in corpus]
    res = gpu_ctx.split_search([im.split_id for im in corpus], plans)
    r = res[0]
    print(f"[fused] K={K}: {_path(r)}")
    assert r.sample_stride == total // grid, _path(r)
    if K <= 1000:  # (at K = 4096 the sample's own target is about the candidate capacity: the repair may run)
        assert r.num_kernel_launches == 2 and r.exact_fallbacks == 0, _path(r)
    else:
        assert r.num_kernel_launches == 2 or r.exact_fallbacks == 1, _path(r)
    _check(res, corpus, plans, f"fused K={K}")


@pytest.mark.gpu
def test_split_without_a_sample_window_takes_two_launches(gpu_ctx, corpus):
    grid = _grid()
    tiny = S.synth_split(W // 2, 99, FRACS, split_id="fused-tiny")  # one window
    gpu_ctx.register_split(tiny)
    try:
        # place the one-window split where no block's chunk begins
        nw = windows(DOCS)
        total = N_SPLITS * nw + 1
        begins = {chunk_begin(total, b, grid) for b in range(grid)}
        pos = next(k for k in range(1, N_SPLITS) if k * nw not in begins)
        imgs = corpus[:pos] + [tiny] + corpus[pos:]
        plans = [_or_plan(im, 100) for im in imgs]
        res = gpu_ctx.split_search([im.split_id for im in imgs], plans)
        r = res[0]
        print(f"[fused] no sample window: {_path(r)}")
        assert r.num_kernel_launches >= 4 and r.sample_stride >= 2 and r.sample_stride != (N_SPLITS * nw + 1) // grid, _path(r)
        _check(res, imgs, plans, "two-launch")
    finally:
        gpu_ctx.unregister_split(tiny.split_id)


def _tie_corpus(split_id, n):
    """Every 64th doc holds the rare term `z` once, in a doc of the same length as every other: more docs share the
    top score than the candidate capacity holds. Half the docs hold the common term `x` (lower scores)."""
    d = np.arange(n, dtype=np.int64)
    lens = np.full(n, 5, dtype=np.int64)
    b = S._Builder(n)
    L = ffi.img_lib()
    fn = np.full(n, L.qwgpu_fieldnorm_to_id(5), dtype=np.uint8)
    body = b.add_field("body", ffi.FIELD_HAS_FREQS | ffi.FIELD_HAS_FIELDNORMS, ffi.TOK_DEFAULT, fn, int(lens.sum()))
    x = np.flatnonzero(d % 2 == 1).astype(np.uint32)
    b.add_term(body, b"x", x, (1 + x % 4).astype(np.uint32))
    z = np.flatnonzero(d % 64 == 0).astype(np.uint32)
    b.add_term(body, b"z", z, np.ones(len(z), dtype=np.uint32))
    return b.finish(split_id)


@pytest.mark.gpu
def test_tie_overflow_takes_the_exact_repair(gpu_ctx):
    grid = _grid()
    imgs = [_tie_corpus(f"fused-tie-{i}", DOCS) for i in range(N_SPLITS)]
    for im in imgs:
        gpu_ctx.register_split(im)
    try:
        plans = [_or_plan(im, 10, terms=("x", "z")) for im in imgs]
        res = gpu_ctx.split_search([im.split_id for im in imgs], plans)
        r = res[0]
        print(f"[fused] tie overflow: {_path(r)}")
        assert r.sample_stride == N_SPLITS * windows(DOCS) // grid, _path(r)
        assert r.exact_fallbacks == 1 and r.radix_passes >= 1, _path(r)
        _check(res, imgs, plans, "tie")
    finally:
        for im in imgs:
            gpu_ctx.unregister_split(im.split_id)


@pytest.mark.gpu
def test_concurrent_fused_calls_match_sequential(gpu_ctx, corpus):
    """Eight host threads issue the same fused call at once: cooperative grids on eight streams, one grid barrier
    each. Run once."""
    ids = [im.split_id for im in corpus]
    plans = [_or_plan(im, 1000) for im in corpus]
    want = gpu_ctx.split_search(ids, plans)
    assert want[0].num_kernel_launches == 2, _path(want[0])
    with ThreadPoolExecutor(8) as ex:
        got = list(ex.map(lambda _: gpu_ctx.split_search(ids, plans), range(8)))
    for t, res in enumerate(got):
        assert res[0].num_kernel_launches == 2, _path(res[0])
        for i, (g, w) in enumerate(zip(res, want)):
            assert g.num_hits == w.num_hits and g.hits == w.hits, f"thread {t} split {i}"
