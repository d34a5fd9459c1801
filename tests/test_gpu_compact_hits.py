"""Hits of plans ranked by `_score` descending alone come back from the device as (doc id, score) pairs and are
expanded to QwHit on the host (qwgpu_format.h QwScoreHit). The expansion must be invisible: every QwHit the library
returns equals, byte for byte, what the same call returns when the plans carry QW_PLAN_FULL_HITS (the device writes
full records). The corpus gives every split a few dozen distinct scores, so that ties straddle the K-th hit at every
K; batches mix compact and full plans, on the BM25-union route and on the generic window route."""
import ctypes as C

import numpy as np
import pytest

from quickwit_b200 import ffi, plan as P, splitgen as S

pytestmark = pytest.mark.gpu

N = 1 << 18  # docs per split: > 16 union windows, so the threshold is sampled
FULL_HITS = 1  # QW_PLAN_FULL_HITS


def _corpus(split_id):
    d = np.arange(N, dtype=np.int64)
    lens = 1 + (d * 7919) % 12
    b = S._Builder(N)
    L = ffi.img_lib()
    fn = np.array([L.qwgpu_fieldnorm_to_id(int(x)) for x in range(13)], dtype=np.uint8)[lens]
    body = b.add_field("body", ffi.FIELD_HAS_FREQS | ffi.FIELD_HAS_FIELDNORMS, ffi.TOK_DEFAULT, fn, int(lens.sum()))
    x = np.flatnonzero(d % 3 != 0).astype(np.uint32)
    b.add_term(body, b"x", x, (1 + x % 3).astype(np.uint32))
    y = np.flatnonzero(d % 5 == 0).astype(np.uint32)
    b.add_term(body, b"y", y, np.ones(len(y), dtype=np.uint32))
    b.add_column("a", ffi.COL_U64, ffi.CARD_FULL, ((d * 2654435761) % 1000).astype(np.uint64), None)
    return b.finish(split_id)


@pytest.fixture(scope="module")
def splits(gpu_ctx):
    imgs = [_corpus(f"compact-{i}") for i in range(3)]
    for img in imgs:
        gpu_ctx.register_split(img)
    yield imgs
    for img in imgs:
        gpu_ctx.unregister_split(img.split_id)


def _plan(img, K, sort=((ffi.SORT_SCORE, ffi.ORDER_DESC, ffi.ABSENT),), full=False):
    root = P.bool_([P.term(img, "body", t, occur=ffi.OCCUR_SHOULD) for t in ("x", "y")])
    plan = P.make_plan(root, K, list(sort))
    if not full:
        return plan
    h = ffi.QwPlanHeader.from_buffer_copy(plan)
    h.reserved |= FULL_HITS
    return bytes(h) + plan[C.sizeof(h):]


def _search(ctx, ids, plans):
    """Seam C, keeping each split's QwHit array as raw bytes and the call's path."""
    L = ffi.lib()
    n = len(ids)
    bufs = [C.create_string_buffer(p, len(p)) for p in plans]
    res = (ffi.SplitResult * n)()
    status = (C.c_int * n)()
    ffi.check(L.qwgpu_split_search(ctx._ctx, n, (C.c_char_p * n)(*[s.encode() for s in ids]),
                                   (C.c_void_p * n)(*[C.addressof(b) for b in bufs]), (C.c_size_t * n)(*[len(p) for p in plans]),
                                   res, status))
    try:
        assert list(status) == [0] * n, L.qwgpu_last_error().decode()
        hits = [C.string_at(res[i].hits, res[i].num_partial_hits * C.sizeof(ffi.QwHit)) for i in range(n)]
        path = (res[0].kernel_mask, res[0].sample_stride, res[0].num_kernel_launches, res[0].exact_fallbacks)
        return hits, [res[i].num_hits for i in range(n)], path
    finally:
        for i in range(n):
            L.qwgpu_split_result_free(C.byref(res[i]))


def _same(ctx, ids, compact_plans, full_plans, union):
    got, got_n, got_path = _search(ctx, ids, compact_plans)
    want, want_n, want_path = _search(ctx, ids, full_plans)
    assert got_n == want_n
    assert got_path == want_path, (got_path, want_path)
    mask, stride, launches, _ = got_path
    assert launches >= 4 and (stride >= 2 or not union)
    assert bool(mask & ffi.KERNEL_UNION) == union, hex(mask)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"split {i}: QwHit bytes differ"
    return got


def _hit_fields(raw):
    return np.frombuffer(raw, dtype=np.dtype([("v1", "<u8"), ("v2", "<u8"), ("doc_id", "<u4"), ("flags", "<u4"),
                                              ("score", "<f4"), ("reserved", "<u4")]))


@pytest.mark.parametrize("K", [1, 10, 1000, 4096])
def test_score_hits_equal_full_records(gpu_ctx, splits, K):
    ids = [img.split_id for img in splits]
    got = _same(gpu_ctx, ids, [_plan(img, K) for img in splits], [_plan(img, K, full=True) for img in splits], union=True)
    # the best score belongs to every doc with tf(x) = 3, y present and length 2 — more docs than any K: the K-th hit
    # ties with docs that did not make the list
    d = np.arange(N)
    top = (d % 3 == 2) & (d % 5 == 0) & (1 + (d * 7919) % 12 == 2)
    assert top.sum() > K
    for raw in got:
        h = _hit_fields(raw)
        assert len(h) == K and (h["score"] == h["score"][0]).all() and top[h["doc_id"]].all()
        assert (h["flags"] == 1).all() and (h["v2"] == 0).all() and (h["reserved"] == 0).all()


def test_batch_mixing_compact_and_full_plans(gpu_ctx, splits):
    ids = [img.split_id for img in splits]
    # BM25-union route: one split's plan keeps full records, the others are compact
    mixed = [_plan(splits[0], 1000), _plan(splits[1], 1000, full=True), _plan(splits[2], 10)]
    full = [_plan(img, k, full=True) for img, k in zip(splits, (1000, 1000, 10))]
    _same(gpu_ctx, ids, mixed, full, union=True)
    # generic route: a column sort in the batch (full records by nature) next to compact _score plans
    by_col = ((ffi.SORT_COLUMN, ffi.ORDER_DESC, 0),)
    mixed = [_plan(splits[0], 1000), _plan(splits[1], 100, sort=by_col), _plan(splits[2], 4096)]
    full = [_plan(splits[0], 1000, full=True), _plan(splits[1], 100, sort=by_col), _plan(splits[2], 4096, full=True)]
    _same(gpu_ctx, ids, mixed, full, union=False)
