"""Host-side mirror of the reference interface for this path (Python twin of the Rust shim a
Quickwit maintainer would write over the C ABI; see INTEGRATION.md).

Names follow the reference:
  * `SearcherContext`      — quickwit-search/src/service.rs:405-498 (owns caches; here: HBM residency)
  * `SearchService.leaf_search(LeafSearchRequest) -> LeafSearchResponse`
                           — quickwit-search/src/service.rs:81,177-203  (seam A)
  * `LambdaLeafSearchInvoker.invoke_leaf_search(LeafSearchRequest) -> [LambdaSingleSplitResult]`
                           — quickwit-search/src/invoker.rs:27-38       (seam B)
  * `leaf_search_single_split` on a compiled plan (seam C, leaf.rs:498-705 step 10c)
All of them call straight into libqwgpu.so; nothing here computes results.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple

from . import ffi
from .splitgen import SplitImage


class SplitSearchResult:
    """Fields of the per-split `LeafSearchResponse` before protobuf encoding."""

    def __init__(self, r: ffi.SplitResult):
        self.num_hits = int(r.num_hits)
        self.hits: List[Tuple[int, int, int, int, float]] = [
            (h.doc_id, h.flags, h.v1, h.v2, h.score) for h in (r.hits[i] for i in range(r.num_partial_hits))]
        self.cells = [(c.count, c.sum_bits, c.min_mapped, c.max_mapped)
                      for c in (r.agg_cells[i] for i in range(r.num_agg_cells))]
        self.gpu_time_us = float(r.gpu_time_us)
        self.main_kernel_us = float(r.main_kernel_us)
        self.exact_fallbacks = int(r.exact_fallbacks)
        self.num_kernel_launches = int(r.num_kernel_launches)
        self.postings_scored = int(r.postings_scored)
        self.algorithmic_bytes = int(r.algorithmic_bytes)
        # the path the call took (per call, the same for every split of the batch)
        self.kernel_mask = int(r.kernel_mask)
        self.window_docs = int(r.window_docs)
        self.sample_stride = int(r.sample_stride)
        self.radix_passes = int(r.radix_passes)
        self.refined = int(r.refined)


class SearcherContext:
    """Owns one `qwgpu_ctx` (one GPU). device=None gives a host-only context (plan compilation,
    merging); any search call on it raises QwGpuError(ENODEVICE) — there is no CPU search path."""

    def __init__(self, device: Optional[int] = 0):
        self._L = ffi.lib()
        self._ctx = C.c_void_p()
        ffi.check(self._L.qwgpu_init(-1 if device is None else device, C.byref(self._ctx)))

    def close(self):
        if self._ctx:
            self._L.qwgpu_shutdown(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- residency (open_index_with_caches + warmup, leaf.rs:210-251,269-472) --------------------
    def register_split(self, img: SplitImage, split_id: Optional[str] = None):
        ffi.check(self._L.qwgpu_split_register(self._ctx, (split_id or img.split_id).encode(), img.ptr, img.nbytes))

    def unregister_split(self, split_id: str):
        ffi.check(self._L.qwgpu_split_unregister(self._ctx, split_id.encode()))

    def resident_bytes(self) -> int:
        return int(self._L.qwgpu_resident_bytes(self._ctx))

    def set_residency_budget(self, nbytes: int):
        """Cap on the split data kept in HBM; registrations beyond it evict the least recently searched splits."""
        ffi.check(self._L.qwgpu_set_residency_budget(self._ctx, nbytes))

    def register_split_async(self, img: SplitImage, split_id: Optional[str] = None):
        """Background upload; `img` must stay alive until wait_split() has returned."""
        ffi.check(self._L.qwgpu_split_register_async(self._ctx, (split_id or img.split_id).encode(), img.ptr, img.nbytes))

    def wait_split(self, split_id: str):
        ffi.check(self._L.qwgpu_split_wait(self._ctx, split_id.encode()))

    def is_resident(self, split_id: str) -> bool:
        return bool(self._L.qwgpu_split_is_resident(self._ctx, split_id.encode()))

    def residency_info(self) -> dict:
        v = [C.c_uint64() for _ in range(4)]
        ffi.check(self._L.qwgpu_residency_info(self._ctx, *[C.byref(x) for x in v]))
        return dict(zip(("resident_bytes", "budget_bytes", "num_splits", "evictions"), (int(x.value) for x in v)))

    # -- seam C -------------------------------------------------------------------------------------
    def split_search(self, split_ids: Sequence[str], plans: Sequence[bytes]) -> List[SplitSearchResult]:
        n = len(split_ids)
        ids = (C.c_char_p * n)(*[s.encode() for s in split_ids])
        bufs = [C.create_string_buffer(p, len(p)) for p in plans]
        pp = (C.c_void_p * n)(*[C.addressof(b) for b in bufs])
        ln = (C.c_size_t * n)(*[len(p) for p in plans])
        res = (ffi.SplitResult * n)()
        status = (C.c_int * n)()
        ffi.check(self._L.qwgpu_split_search(self._ctx, n, ids, pp, ln, res, status))
        try:
            for i in range(n):
                if status[i] != 0:
                    raise ffi.QwGpuError(status[i], self._L.qwgpu_last_error().decode("utf-8", "replace"))
            return [SplitSearchResult(res[i]) for i in range(n)]
        finally:
            for i in range(n):
                self._L.qwgpu_split_result_free(C.byref(res[i]))

    # -- seam A / B -----------------------------------------------------------------------------------
    def _bytes_call(self, fn, req: bytes) -> bytes:
        buf = C.create_string_buffer(req, len(req))
        out, n = C.c_void_p(), C.c_size_t()
        ffi.check(fn(self._ctx, C.addressof(buf), len(req), C.byref(out), C.byref(n)))
        return ffi.take_bytes(out, n.value)

    def leaf_search(self, leaf_search_request: bytes) -> bytes:
        """SearchService::leaf_search: LeafSearchRequest bytes -> LeafSearchResponse bytes."""
        return self._bytes_call(self._L.qwgpu_leaf_search, leaf_search_request)

    # -- collectives (one process per GPU) ----------------------------------------------------------------
    @staticmethod
    def comm_unique_id() -> bytes:
        """Rank 0: the 128-byte NCCL unique id to hand to the other ranks."""
        buf = C.create_string_buffer(128)
        ffi.check(ffi.lib().qwgpu_comm_unique_id(C.addressof(buf)))
        return buf.raw

    def comm_init(self, unique_id: bytes, rank: int, world: int, all_split_ids: Sequence[str]):
        """Builds this context's NCCL communicator and the global split table (tie-break ranks)."""
        idb = C.create_string_buffer(unique_id, 128)
        ffi.check(self._L.qwgpu_comm_init(self._ctx, C.addressof(idb), rank, world))
        n = len(all_split_ids)
        arr = (C.c_char_p * n)(*[s.encode() for s in all_split_ids])
        ffi.check(self._L.qwgpu_comm_set_split_table(self._ctx, n, arr))

    def comm_init_lane(self, lane: int, unique_id: bytes, rank: int, world: int):
        """One more communicator on this context (its own unique id): concurrent collective searches take one
        lane each, the same request-to-lane assignment on every rank."""
        idb = C.create_string_buffer(unique_id, 128)
        ffi.check(self._L.qwgpu_comm_init_lane(self._ctx, lane, C.addressof(idb), rank, world))

    def leaf_search_allgather(self, leaf_search_request: bytes, lane: int = 0) -> bytes:
        """Collective: leaf_search on this rank's splits + the device-side all-gather / merge that stands in
        for the root merge; every rank returns the merged LeafSearchResponse."""
        L = self._L
        buf = C.create_string_buffer(leaf_search_request, len(leaf_search_request))
        out, n = C.c_void_p(), C.c_size_t()
        ffi.check(L.qwgpu_leaf_search_allgather_lane(self._ctx, lane, C.addressof(buf), len(leaf_search_request), C.byref(out), C.byref(n)))
        return ffi.take_bytes(out, n.value)

    def invoke_leaf_search(self, leaf_search_request: bytes) -> bytes:
        """LambdaLeafSearchInvoker::invoke_leaf_search -> LambdaSearchResponses bytes."""
        return self._bytes_call(self._L.qwgpu_invoke_leaf_search, leaf_search_request)


def compile_plan(img: SplitImage, search_request_pb: bytes, doc_mapper_json: str, split_id: str = "") -> bytes:
    """doc_mapper.query + make_collector_for_split for one split (host only)."""
    L = ffi.lib()
    buf = C.create_string_buffer(search_request_pb, len(search_request_pb))
    out, n = C.c_void_p(), C.c_size_t()
    ffi.check(L.qwgpu_compile_plan(img.ptr, img.nbytes, (split_id or img.split_id).encode(), C.addressof(buf),
                                   len(search_request_pb), doc_mapper_json.encode(), C.byref(out), C.byref(n)))
    return ffi.take_bytes(out, n.value)


def optimize_leaf_request(leaf_search_request_pb: bytes) -> list:
    """CanSplitDoBetter::optimize + metadata-count detection for every split of a LeafSearchRequest
    (leaf.rs:1072-1242, root.rs:665-686): [{"split_id", "max_hits", "hits_disabled", "metadata_count"}]
    in the reference's processing order. Host only."""
    import json
    L = ffi.lib()
    buf = C.create_string_buffer(leaf_search_request_pb, len(leaf_search_request_pb))
    out, n = C.c_void_p(), C.c_size_t()
    ffi.check(L.qwgpu_optimize_leaf_request(C.addressof(buf), len(leaf_search_request_pb), C.byref(out), C.byref(n)))
    return json.loads(ffi.take_bytes(out, n.value))


def parse_split_footer(tail: bytes, split_file_len: int) -> dict:
    """BundleStorageFileOffsets + HotDirectoryMeta of a `.split` file from its last bytes
    (bundle_storage.rs:92-174, hot_directory.rs:40-80): where the tantivy files and the hotcache lie. Host only."""
    import json
    L = ffi.lib()
    buf = C.create_string_buffer(tail, len(tail))
    out, n = C.c_void_p(), C.c_size_t()
    ffi.check(L.qwgpu_parse_split_footer(C.addressof(buf), len(tail), split_file_len, C.byref(out), C.byref(n)))
    return json.loads(ffi.take_bytes(out, n.value))


def merge_leaf_responses(search_request_pb: bytes, responses: Sequence[bytes]) -> bytes:
    """merge_leaf_responses / QuickwitCollector::merge_fruits (collector.rs:832-974)."""
    L = ffi.lib()
    n = len(responses)
    rb = C.create_string_buffer(search_request_pb, len(search_request_pb))
    bufs = [C.create_string_buffer(r, max(len(r), 1)) for r in responses]
    pp = (C.c_void_p * n)(*[C.addressof(b) for b in bufs])
    ln = (C.c_size_t * n)(*[len(r) for r in responses])
    out, m = C.c_void_p(), C.c_size_t()
    ffi.check(L.qwgpu_merge_leaf_responses(C.addressof(rb), len(search_request_pb), n, pp, ln, C.byref(out), C.byref(m)))
    return ffi.take_bytes(out, m.value)


def finalize_aggregation(aggregation_request_json: str, intermediate: bytes) -> str:
    """finalize_aggregation (root.rs:1105-1135): intermediate bytes -> final aggregation JSON."""
    L = ffi.lib()
    ib = C.create_string_buffer(intermediate, max(len(intermediate), 1))
    out = C.c_void_p()
    ffi.check(L.qwgpu_finalize_aggregation(aggregation_request_json.encode(), C.addressof(ib), len(intermediate), C.byref(out)))
    try:
        return C.string_at(out).decode()
    finally:
        L.qwgpu_buf_free(out)


def decode_spans(intermediate: bytes) -> List[Tuple[bytes, int]]:
    """find_trace_ids result bytes (postcard `Vec<Span>`: varint length, then per span the 16 trace-id bytes and
    the zigzag varint of the i64 timestamp in ns) -> [(trace_id, span_timestamp_ns), ...] in wire order."""
    pos = 0

    def varint() -> int:
        nonlocal pos
        v = sh = 0
        while True:
            if pos >= len(intermediate):
                raise ValueError("truncated varint")
            b = intermediate[pos]
            pos += 1
            v |= (b & 0x7F) << sh
            if not b & 0x80:
                return v
            sh += 7

    spans = []
    for _ in range(varint()):
        if len(intermediate) - pos < 16:
            raise ValueError("truncated span")
        tid = bytes(intermediate[pos:pos + 16])
        pos += 16
        z = varint()
        spans.append((tid, (z >> 1) ^ -(z & 1)))
    if pos != len(intermediate):
        raise ValueError("trailing bytes")
    return spans


def build_leaf_response(img: SplitImage, search_request_pb: bytes, doc_mapper_json: str, num_hits: int,
                        hits: Sequence[Tuple[int, int, int, int, float]], cells: Sequence[Tuple[int, int, int, int]],
                        split_id: str = "") -> bytes:
    """QuickwitSegmentCollector::harvest for a seam-C result: hits are (doc_id, flags, v1, v2, score),
    cells are (count, sum_bits, min_mapped, max_mapped). Returns LeafSearchResponse bytes."""
    L = ffi.lib()
    rb = C.create_string_buffer(search_request_pb, len(search_request_pb))
    harr = (ffi.QwHit * max(len(hits), 1))()
    for i, (doc, flags, v1, v2, score) in enumerate(hits):
        harr[i].doc_id, harr[i].flags, harr[i].v1, harr[i].v2, harr[i].score = doc, flags, v1, v2, score
    carr = (ffi.QwAggCell * max(len(cells), 1))()
    for i, (cnt, s, mn, mx) in enumerate(cells):
        carr[i].count, carr[i].sum_bits, carr[i].min_mapped, carr[i].max_mapped = cnt, s, mn, mx
    out, n = C.c_void_p(), C.c_size_t()
    ffi.check(L.qwgpu_build_leaf_response(img.ptr, img.nbytes, (split_id or img.split_id).encode(), C.addressof(rb),
                                          len(search_request_pb), doc_mapper_json.encode(), num_hits, harr, len(hits),
                                          carr, len(cells), C.byref(out), C.byref(n)))
    return ffi.take_bytes(out, n.value)


# ---- multi-GPU partial exchange (SURVEY.md §8e): one fixed-size all-gather stands in for the root merge
def partial_size(search_request_pb: bytes) -> int:
    L = ffi.lib()
    rb = C.create_string_buffer(search_request_pb, len(search_request_pb))
    n = C.c_uint64()
    ffi.check(L.qwgpu_partial_size(C.addressof(rb), len(search_request_pb), C.byref(n)))
    return int(n.value)


def response_to_partial(search_request_pb: bytes, leaf_response: bytes, out_ptr: int, nbytes: int) -> None:
    """Packs a rank's LeafSearchResponse into the fixed-size partial at `out_ptr` (host memory)."""
    L = ffi.lib()
    rb = C.create_string_buffer(search_request_pb, len(search_request_pb))
    lb = C.create_string_buffer(leaf_response, max(len(leaf_response), 1))
    ffi.check(L.qwgpu_response_to_partial(C.addressof(rb), len(search_request_pb), C.addressof(lb), len(leaf_response), out_ptr, nbytes))


def merge_partials(search_request_pb: bytes, n_ranks: int, gathered_ptr: int, partial_bytes: int) -> bytes:
    """merge_leaf_responses over the all-gathered partials of every rank -> LeafSearchResponse bytes."""
    L = ffi.lib()
    rb = C.create_string_buffer(search_request_pb, len(search_request_pb))
    out, n = C.c_void_p(), C.c_size_t()
    ffi.check(L.qwgpu_merge_partials(C.addressof(rb), len(search_request_pb), n_ranks, gathered_ptr, partial_bytes, C.byref(out), C.byref(n)))
    return ffi.take_bytes(out, n.value)
