//! `extern "C"` surface of libqwgpu (include/qwgpu.h). Plain pointers and sizes; every buffer the library returns is
//! malloc'ed by it and released with `qwgpu_buf_free`.

use std::ffi::{CStr, c_char, c_void};

use quickwit_search::SearchError;

#[repr(C)]
pub struct QwgpuCtx {
    _private: [u8; 0],
}

pub const QWGPU_OK: i32 = 0;
pub const QWGPU_EINTERNAL: i32 = -1;
pub const QWGPU_EINVALID_QUERY: i32 = -2;
pub const QWGPU_EINVALID_AGG: i32 = -3;
pub const QWGPU_EINVALID_ARG: i32 = -4;
pub const QWGPU_ENODEVICE: i32 = -5;
pub const QWGPU_ENOTFOUND: i32 = -6;
pub const QWGPU_EUNSUPPORTED: i32 = -7;

#[link(name = "qwgpu")]
unsafe extern "C" {
    pub fn qwgpu_last_error() -> *const c_char;
    pub fn qwgpu_buf_free(buf: *mut c_void);

    pub fn qwgpu_init(device: i32, out: *mut *mut QwgpuCtx) -> i32;
    pub fn qwgpu_shutdown(ctx: *mut QwgpuCtx);

    pub fn qwgpu_split_register(ctx: *mut QwgpuCtx, split_id: *const c_char, img: *const u8, img_len: u64) -> i32;
    pub fn qwgpu_split_register_async(ctx: *mut QwgpuCtx, split_id: *const c_char, img: *const u8, img_len: u64) -> i32;
    pub fn qwgpu_split_wait(ctx: *mut QwgpuCtx, split_id: *const c_char) -> i32;
    pub fn qwgpu_split_unregister(ctx: *mut QwgpuCtx, split_id: *const c_char) -> i32;
    pub fn qwgpu_split_is_resident(ctx: *mut QwgpuCtx, split_id: *const c_char) -> i32;
    pub fn qwgpu_set_residency_budget(ctx: *mut QwgpuCtx, bytes: u64) -> i32;
    pub fn qwgpu_set_max_hits(ctx: *mut QwgpuCtx, max_hits: u32) -> i32;
    pub fn qwgpu_set_predicate_cache_budget(ctx: *mut QwgpuCtx, bytes: u64) -> i32;
    pub fn qwgpu_predicate_cache_info(ctx: *mut QwgpuCtx, budget_bytes: *mut u64, used_bytes: *mut u64, entries: *mut u64,
                                      hits: *mut u64, misses: *mut u64, fills: *mut u64, evictions: *mut u64) -> i32;
    pub fn qwgpu_resident_bytes(ctx: *mut QwgpuCtx) -> u64;

    /// prost-encoded `LeafSearchRequest` in, prost-encoded `LeafSearchResponse` out (seam A).
    pub fn qwgpu_leaf_search(ctx: *mut QwgpuCtx, req: *const u8, req_len: usize, resp: *mut *mut u8, resp_len: *mut usize) -> i32;
    /// prost-encoded `LeafSearchRequest` in, prost-encoded `LambdaSearchResponses` out (seam B).
    pub fn qwgpu_invoke_leaf_search(ctx: *mut QwgpuCtx, req: *const u8, req_len: usize, resp: *mut *mut u8, resp_len: *mut usize) -> i32;

    pub fn qwgpu_merge_leaf_responses(
        search_request: *const u8, search_request_len: usize, n: u32, resps: *const *const u8, resp_lens: *const usize,
        merged: *mut *mut u8, merged_len: *mut usize,
    ) -> i32;
    pub fn qwgpu_finalize_aggregation(aggregation_request_json: *const c_char, intermediate: *const u8, intermediate_len: usize, json_out: *mut *mut c_char) -> i32;

    pub fn qwgpu_parse_split_footer(tail: *const u8, tail_len: u64, split_file_len: u64, json_out: *mut *mut u8, json_len: *mut usize) -> i32;
}

/// Thread-local message of the last failed call on this thread.
pub fn last_error() -> String {
    unsafe {
        let p = qwgpu_last_error();
        if p.is_null() { String::new() } else { CStr::from_ptr(p).to_string_lossy().into_owned() }
    }
}

/// Return codes onto `SearchError` (quickwit-search/src/error.rs:32-53). `QWGPU_EUNSUPPORTED` is deterministic for
/// a request: the caller routes such requests to the CPU searcher, the library never falls back by itself.
pub fn map_error(rc: i32) -> SearchError {
    let msg = last_error();
    match rc {
        QWGPU_EINVALID_QUERY => SearchError::InvalidQuery(msg),
        QWGPU_EINVALID_AGG => SearchError::InvalidAggregationRequest(msg),
        QWGPU_EINVALID_ARG => SearchError::InvalidArgument(msg),
        QWGPU_ENODEVICE | QWGPU_ENOTFOUND => SearchError::Unavailable(msg),
        QWGPU_EUNSUPPORTED => SearchError::Internal(format!("unsupported on the GPU path: {msg}")),
        _ => SearchError::Internal(msg),
    }
}

/// Runs a "bytes in, malloc'ed bytes out" entry point and copies the result into a `Vec`.
pub unsafe fn bytes_call(
    f: unsafe extern "C" fn(*mut QwgpuCtx, *const u8, usize, *mut *mut u8, *mut usize) -> i32,
    ctx: *mut QwgpuCtx,
    request: &[u8],
) -> Result<Vec<u8>, SearchError> {
    let (mut out, mut len) = (std::ptr::null_mut::<u8>(), 0usize);
    let rc = unsafe { f(ctx, request.as_ptr(), request.len(), &mut out, &mut len) };
    if rc != QWGPU_OK {
        return Err(map_error(rc));
    }
    let bytes = unsafe { std::slice::from_raw_parts(out, len) }.to_vec();
    unsafe { qwgpu_buf_free(out as *mut c_void) };
    Ok(bytes)
}
