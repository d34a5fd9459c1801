"""k_window's boolean program at the limits it was sized for, against bool_ref's restatement (built from the corpus
arrays, never the image) and the oracle, bit for bit: doc ids, sort values, f32 score bits, num_hits.

Every call asserts that it ran on k_window (KERNEL_WINDOW, neither KERNEL_UNION nor KERNEL_DRIVER, a pure BM25 OR in
a mixed batch included) at the window size its case targets (restated from the shared-memory layout by
bool_ref.window_docs, checked on the CPU by test_bool_limits_host.py), and that a plan asking for hits sampled its
threshold. The cases (test_bool_limits_host.py): four bool levels, scored and unscored; every minimum_should_match
at levels 0 and 3; the weights around IF_BITS_FROM_SCORE; 64 terms, 96 instructions, two scored fields and 16
columns, as a pure OR and as a tree; one over each limit (refused, then the context still answers); the staging
regimes of phase 2 at every window size; a batch over two splits of plans of 1..4 levels and a pure OR."""
import time

import pytest
import torch

from quickwit_b200 import ffi
from helpers import assert_same
from regex_ref import oracle_search
import bool_corpora as BC
import bool_ref as B
import test_bool_limits_host as H

pytestmark = pytest.mark.gpu

REACHED = set()


@pytest.fixture(scope="module")
def splits(gpu_ctx):
    t = time.time()
    main, small = BC.main_split(), BC.small_split()
    print(f"[bool limits] splits built in {time.time() - t:.1f} s")
    for sp in (main, small):
        gpu_ctx.register_split(sp.img)
    yield main, small
    for sp in (main, small):
        gpu_ctx.unregister_split(sp.split_id)


def run(ctx, label, W, items):
    plans = [B.plan(sp, q, sort, K, sa) for sp, q, sort, K, sa in items]
    res = ctx.split_search([it[0].split_id for it in items], plans)
    for (sp, q, sort, K, sa), r, pl in zip(items, res, plans):
        tag = f"{label} {sp.split_id} {q!r} sort={sort.keys} K={K} kernel_mask={r.kernel_mask:#x} W={r.window_docs}"
        assert r.kernel_mask & ffi.KERNEL_WINDOW and not r.kernel_mask & (ffi.KERNEL_UNION | ffi.KERNEL_DRIVER), tag
        assert r.window_docs == W, tag
        if K and sp.n > 8 * 2 * W:
            assert r.sample_stride > 1, tag
        assert_same(r, oracle_search(sp.img, pl), ctx=tag)
        B.check(r, sp, q, sort, K, sa, ctx=tag)
    REACHED.add(W)
    return res


def test_shared_memory_is_what_the_layout_assumes():
    """The window sizes are restated for a 227 KB opt-in per block."""
    props = torch.cuda.get_device_properties(0)
    assert props.shared_memory_per_block_optin == B.H100_SMEM_OPTIN, props.shared_memory_per_block_optin


@pytest.mark.parametrize("group", ["depth", "msm", "weights", "limits", "staging", "batch"])
def test_calls(gpu_ctx, splits, group):
    main, small = splits
    calls = {"depth": H.depth_calls, "msm": H.msm_calls, "weights": H.weight_calls, "limits": H.limit_calls,
             "staging": H.regime_calls}.get(group)
    if calls is None:
        b = H.batch_call(main, small)
        calls = lambda m: [(b[0][0], b[0][1], H.with_search_after(list(b[0][2])))]
    for label, W, items in calls(main):
        run(gpu_ctx, label, W, items)


def test_refusals_leave_the_context_working(gpu_ctx, splits):
    main, _ = splits
    ok_label, ok_W, ok_items = H.depth_calls(main)[0]
    for label, item, msg in H.refusals(main):
        with pytest.raises(ffi.QwGpuError) as e:
            gpu_ctx.split_search([item[0].split_id], [B.plan(*item)])
        assert e.value.code == ffi.EUNSUPPORTED and msg in str(e.value), (label, str(e.value))
        run(gpu_ctx, f"after {label}: {ok_label}", ok_W, ok_items)


def test_every_window_size_was_reached():
    assert REACHED == set(BC.WINDOWS), sorted(REACHED)
