"""ctypes binding of libqwgpu.so (include/qwgpu.h) — the stub a host language writes over the C ABI.

This is the Python twin of the Rust `extern "C"` block shown in INTEGRATION.md. It holds no
logic: structs mirror include/qwgpu_format.h field for field.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("QWGPU_LIB") or os.path.join(_HERE, "libqwgpu.so")  # QWGPU_LIB: development builds

OK = 0
EINTERNAL, EINVALID_QUERY, EINVALID_AGG, EINVALID_ARG, ENODEVICE, ENOTFOUND, EUNSUPPORTED = (
    -1, -2, -3, -4, -5, -6, -7)

# qwgpu_format.h enums
FIELD_HAS_FREQS, FIELD_HAS_FIELDNORMS, FIELD_HAS_POSITIONS = 1, 2, 4
TOK_RAW, TOK_DEFAULT = 0, 1
COL_U64, COL_I64, COL_F64, COL_BOOL, COL_DATETIME, COL_STR, COL_BYTES = range(7)
CARD_FULL, CARD_OPTIONAL, CARD_MULTI = range(3)
NODE_TERM, NODE_RANGE, NODE_BOOL, NODE_ALL, NODE_NONE, NODE_EXISTS, NODE_PHRASE = 1, 2, 3, 4, 5, 6, 7
NODE_PHRASE_PREFIX = 8
MAX_PHRASE_TERMS, MAX_PREFIX_EXPANSIONS = 8, 1024
OCCUR_MUST, OCCUR_SHOULD, OCCUR_MUST_NOT, OCCUR_FILTER = range(4)
SORT_NONE, SORT_DOCID, SORT_SCORE, SORT_COLUMN = range(4)
ORDER_ASC, ORDER_DESC = 0, 1
AGG_TERMS, AGG_HISTOGRAM, AGG_RANGE, AGG_STATS, AGG_TRACE_IDS = 1, 2, 3, 4, 5
ABSENT = 0xFFFFFFFF
# qwgpu_split_result.kernel_mask (qwgpu.h)
KERNEL_UNION, KERNEL_DRIVER, KERNEL_AGGSCAN, KERNEL_WINDOW, KERNEL_PHRASE = 1, 2, 4, 8, 16
KERNEL_TRACE_SELECT, KERNEL_TRACE_REPLAY = 32, 64
PLAN_MAGIC = 0x4E4C5051
MAX_AGG_RANGES = 16


class QwImgHeader(C.Structure):
    _fields_ = [("magic", C.c_uint64), ("version", C.c_uint32), ("num_docs", C.c_uint32),
                ("num_fields", C.c_uint32), ("num_terms", C.c_uint32), ("num_columns", C.c_uint32),
                ("reserved0", C.c_uint32), ("fields_off", C.c_uint64), ("terms_off", C.c_uint64),
                ("term_bytes_off", C.c_uint64), ("term_bytes_len", C.c_uint64),
                ("columns_off", C.c_uint64), ("strings_off", C.c_uint64), ("strings_len", C.c_uint64),
                ("data_off", C.c_uint64), ("data_len", C.c_uint64), ("total_len", C.c_uint64),
                ("reserved1", C.c_uint64 * 3)]


class QwImgField(C.Structure):
    _fields_ = [("name_off", C.c_uint32), ("name_len", C.c_uint32), ("flags", C.c_uint32),
                ("tokenizer", C.c_uint32), ("total_num_tokens", C.c_uint64),
                ("fieldnorm_off", C.c_uint64), ("first_term", C.c_uint32), ("num_terms", C.c_uint32),
                ("reserved", C.c_uint64)]


class QwImgTerm(C.Structure):
    _fields_ = [("field_id", C.c_uint32), ("bytes_off", C.c_uint32), ("bytes_len", C.c_uint32),
                ("doc_freq", C.c_uint32), ("num_blocks", C.c_uint32), ("win_shift", C.c_uint32),
                ("skip_off", C.c_uint64), ("data_off", C.c_uint64), ("data_len", C.c_uint64),
                ("widx_off", C.c_uint64), ("tf_len", C.c_uint64), ("fn_len", C.c_uint64),
                ("sub_off", C.c_uint64), ("pos_off", C.c_uint64), ("pidx_off", C.c_uint64)]


class QwImgColumn(C.Structure):
    _fields_ = [("name_off", C.c_uint32), ("name_len", C.c_uint32), ("type", C.c_uint32),
                ("cardinality", C.c_uint32), ("min_value", C.c_uint64), ("max_value", C.c_uint64),
                ("gcd", C.c_uint64), ("num_vals", C.c_uint64), ("bits", C.c_uint32),
                ("dict_num_terms", C.c_uint32), ("values_off", C.c_uint64), ("values_len", C.c_uint64),
                ("index_off", C.c_uint64), ("index_len", C.c_uint64), ("dict_off", C.c_uint64),
                ("dict_len", C.c_uint64), ("reserved", C.c_uint64)]


class QwHit(C.Structure):
    _fields_ = [("v1", C.c_uint64), ("v2", C.c_uint64), ("doc_id", C.c_uint32),
                ("flags", C.c_uint32), ("score", C.c_float), ("reserved", C.c_uint32)]


class QwAggCell(C.Structure):
    _fields_ = [("count", C.c_uint64), ("sum_bits", C.c_uint64),
                ("min_mapped", C.c_uint64), ("max_mapped", C.c_uint64)]


class QwPlanNode(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("occur", C.c_uint32), ("boost", C.c_float),
                ("first_child", C.c_uint32), ("num_children", C.c_uint32),
                ("min_should_match", C.c_uint32), ("term_ord", C.c_uint32),
                ("field_id", C.c_uint32), ("bm25_weight", C.c_float), ("column", C.c_uint32),
                ("lo", C.c_uint64), ("hi", C.c_uint64)]


class QwSortSpec(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("order", C.c_uint32), ("column", C.c_uint32),
                ("reserved", C.c_uint32)]


class QwSearchAfter(C.Structure):
    _fields_ = [("present", C.c_uint32), ("has_v1", C.c_uint32), ("has_v2", C.c_uint32),
                ("compare_on_equal", C.c_uint32), ("precomp_order", C.c_int32),
                ("doc_id", C.c_uint32), ("v1", C.c_uint64), ("v2", C.c_uint64)]


class QwAggNode(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("parent", C.c_uint32), ("first_child", C.c_uint32),
                ("num_children", C.c_uint32), ("column", C.c_uint32), ("num_buckets", C.c_uint32),
                ("interval", C.c_double), ("offset", C.c_double), ("base_pos", C.c_int64),
                ("has_bounds", C.c_uint32), ("num_ranges", C.c_uint32),
                ("bound_min", C.c_double), ("bound_max", C.c_double),
                ("range_from", C.c_uint64 * MAX_AGG_RANGES), ("range_to", C.c_uint64 * MAX_AGG_RANGES),
                ("has_missing", C.c_uint32), ("reserved", C.c_uint32), ("missing_value", C.c_uint64)]


class QwPlanHeader(C.Structure):
    _fields_ = [("magic", C.c_uint32), ("version", C.c_uint32), ("num_nodes", C.c_uint32),
                ("num_aggs", C.c_uint32), ("max_hits", C.c_uint32), ("scoring", C.c_uint32),
                ("count_only", C.c_uint32), ("reserved", C.c_uint32),
                ("sort", QwSortSpec * 2), ("search_after", QwSearchAfter)]


class SplitResult(C.Structure):
    _fields_ = [("num_hits", C.c_uint64), ("num_partial_hits", C.c_uint32),
                ("num_agg_cells", C.c_uint32), ("hits", C.POINTER(QwHit)),
                ("agg_cells", C.POINTER(QwAggCell)), ("gpu_time_us", C.c_float),
                ("main_kernel_us", C.c_float), ("num_kernel_launches", C.c_uint32),
                ("exact_fallbacks", C.c_uint32), ("postings_scored", C.c_uint64),
                ("algorithmic_bytes", C.c_uint64), ("kernel_mask", C.c_uint32),
                ("window_docs", C.c_uint32), ("sample_stride", C.c_uint32),
                ("radix_passes", C.c_uint32), ("refined", C.c_uint32)]


class SynthSpec(C.Structure):
    _fields_ = [("num_docs", C.c_uint32), ("split_ord", C.c_uint32), ("seed", C.c_uint64),
                ("num_terms", C.c_uint32), ("term_fracs", C.POINTER(C.c_double)),
                ("ts_start_secs", C.c_int64), ("ts_span_secs", C.c_uint32),
                ("num_tenants", C.c_uint32), ("msg_vocab", C.c_uint32), ("reserved", C.c_uint32)]


class QwGpuError(RuntimeError):
    """Mirrors quickwit_search::SearchError (quickwit-search/src/error.rs:32-53)."""

    def __init__(self, code: int, msg: str):
        super().__init__(f"[{code}] {msg}")
        self.code = code
        self.msg = msg


_lib = None


def lib() -> C.CDLL:
    """Loads libqwgpu.so; raises loudly when the extension has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU fallback for the search path)")
    L = C.CDLL(LIB_PATH)
    vp, cp, u8p = C.c_void_p, C.c_char_p, C.POINTER(C.c_uint8)
    u32, u64, sz = C.c_uint32, C.c_uint64, C.c_size_t
    missing = []

    def bind(name, argtypes=None, restype=C.c_int):
        try:
            fn = getattr(L, name)
        except AttributeError:
            missing.append(name)
            return
        if argtypes is not None:
            fn.argtypes = argtypes
        fn.restype = restype

    bind("qwgpu_last_error", [], cp)
    bind("qwgpu_version", [], cp)
    bind("qwgpu_buf_free", [vp], None)
    bind("qwgpu_init", [C.c_int, C.POINTER(vp)])
    bind("qwgpu_shutdown", [vp], None)
    bind("qwgpu_split_register", [vp, cp, vp, u64])
    bind("qwgpu_split_unregister", [vp, cp])
    bind("qwgpu_resident_bytes", [vp], u64)
    bind("qwgpu_set_residency_budget", [vp, u64])
    bind("qwgpu_split_register_async", [vp, cp, vp, u64])
    bind("qwgpu_split_wait", [vp, cp])
    bind("qwgpu_residency_info", [vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)])
    bind("qwgpu_split_is_resident", [vp, cp])
    bind("qwgpu_leaf_search", [vp, vp, sz, C.POINTER(vp), C.POINTER(sz)])
    bind("qwgpu_invoke_leaf_search", [vp, vp, sz, C.POINTER(vp), C.POINTER(sz)])
    bind("qwgpu_compile_plan", [vp, u64, cp, vp, sz, cp, C.POINTER(vp), C.POINTER(sz)])
    bind("qwgpu_split_search", [vp, u32, C.POINTER(cp), C.POINTER(vp), C.POINTER(sz),
                                C.POINTER(SplitResult), C.POINTER(C.c_int)])
    bind("qwgpu_split_result_free", [C.POINTER(SplitResult)], None)
    bind("qwgpu_build_leaf_response", [vp, u64, cp, vp, sz, cp, u64, vp, u32, vp, u32, C.POINTER(vp), C.POINTER(sz)])
    bind("qwgpu_merge_leaf_responses", [vp, sz, u32, C.POINTER(vp), C.POINTER(sz),
                                        C.POINTER(vp), C.POINTER(sz)])
    bind("qwgpu_optimize_leaf_request", [vp, sz, C.POINTER(vp), C.POINTER(sz)])
    bind("qwgpu_parse_split_footer", [vp, u64, u64, C.POINTER(vp), C.POINTER(sz)])
    bind("qwgpu_finalize_aggregation", [cp, vp, sz, C.POINTER(vp)])
    bind("qwgpu_partial_size", [vp, sz, C.POINTER(u64)])
    bind("qwgpu_response_to_partial", [vp, sz, vp, sz, vp, u64])
    bind("qwgpu_merge_partials", [vp, sz, u32, vp, u64, C.POINTER(vp), C.POINTER(sz)])
    bind("qwgpu_comm_unique_id", [vp])
    bind("qwgpu_comm_init", [vp, vp, C.c_int, C.c_int])
    bind("qwgpu_comm_set_split_table", [vp, u32, C.POINTER(cp)])
    bind("qwgpu_comm_destroy", [vp], None)
    bind("qwgpu_leaf_search_allgather", [vp, vp, sz, C.POINTER(vp), C.POINTER(sz)])
    bind("qwgpu_comm_init_lane", [vp, u32, vp, C.c_int, C.c_int])
    bind("qwgpu_leaf_search_allgather_lane", [vp, u32, vp, sz, C.POINTER(vp), C.POINTER(sz)])
    bind("qwgpu_imgb_new", [u32], vp)
    bind("qwgpu_imgb_free", [vp], None)
    bind("qwgpu_imgb_add_field", [vp, cp, u32, u32, vp, u64])
    bind("qwgpu_imgb_add_term", [vp, u32, vp, u32, vp, vp, u32])
    bind("qwgpu_imgb_add_term_positions", [vp, u32, vp, u32, vp, vp, u32, vp, u64])
    bind("qwgpu_imgb_add_column", [vp, cp, u32, u32, vp, u64, vp, vp, vp, u32])
    bind("qwgpu_imgb_finish", [vp, C.POINTER(vp), C.POINTER(u64)])
    bind("qwgpu_synth_split", [C.POINTER(SynthSpec), C.POINTER(vp), C.POINTER(u64)])
    bind("qwgpu_bm25_weight", [u64, u64, C.c_float], C.c_float)
    bind("qwgpu_bm25_phrase_weight", [vp, u32, u64, C.c_float], C.c_float)
    bind("qwgpu_fieldnorm_to_id", [u32], C.c_uint8)
    bind("qwgpu_id_to_fieldnorm", [C.c_uint8], u32)
    if missing and not os.environ.get("QWGPU_DEV_PARTIAL"):
        raise ImportError(f"{LIB_PATH} does not export: {', '.join(missing)} (stale build?)")
    _lib = L
    return L


_img_lib = None


def img_lib():
    """libqwimg.so: the host-only split-image writer (same qwgpu_imgb_* / qwgpu_synth_split entry points as
    libqwgpu.so, built from the same sources, no CUDA). Corpus generation never maps the GPU library."""
    global _img_lib
    if _img_lib is None:
        L = C.CDLL(os.environ.get("QWIMG_LIB") or os.path.join(_HERE, "libqwimg.so"))
        vp, cp, u32, u64 = C.c_void_p, C.c_char_p, C.c_uint32, C.c_uint64
        for name, argtypes, restype in [
                ("qwgpu_last_error", [], cp), ("qwgpu_buf_free", [vp], None),
                ("qwgpu_imgb_new", [u32], vp), ("qwgpu_imgb_free", [vp], None),
                ("qwgpu_imgb_add_field", [vp, cp, u32, u32, vp, u64], C.c_int),
                ("qwgpu_imgb_add_term", [vp, u32, vp, u32, vp, vp, u32], C.c_int),
                ("qwgpu_imgb_add_term_positions", [vp, u32, vp, u32, vp, vp, u32, vp, u64], C.c_int),
                ("qwgpu_imgb_add_column", [vp, cp, u32, u32, vp, u64, vp, vp, vp, u32], C.c_int),
                ("qwgpu_imgb_finish", [vp, C.POINTER(vp), C.POINTER(u64)], C.c_int),
                ("qwgpu_synth_split", [C.POINTER(SynthSpec), C.POINTER(vp), C.POINTER(u64)], C.c_int),
                ("qwgpu_bm25_weight", [u64, u64, C.c_float], C.c_float),
                ("qwgpu_bm25_phrase_weight", [vp, u32, u64, C.c_float], C.c_float),
                ("qwgpu_fieldnorm_to_id", [u32], C.c_uint8), ("qwgpu_id_to_fieldnorm", [C.c_uint8], u32)]:
            fn = getattr(L, name)
            fn.argtypes, fn.restype = argtypes, restype
        _img_lib = L
    return _img_lib


def img_check(rc: int) -> int:
    if rc < 0:
        raise QwGpuError(rc, img_lib().qwgpu_last_error().decode("utf-8", "replace"))
    return rc


def check(rc: int) -> int:
    if rc < 0:
        raise QwGpuError(rc, lib().qwgpu_last_error().decode("utf-8", "replace"))
    return rc


def take_bytes(ptr: C.c_void_p, n: int) -> bytes:
    """Copies a library-owned buffer into Python bytes and frees it."""
    try:
        return C.string_at(ptr, n)
    finally:
        lib().qwgpu_buf_free(ptr)
