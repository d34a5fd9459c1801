//! Owning wrapper of a `qwgpu_ctx` (one per GPU). Every entry point of the library is re-entrant on one context
//! (a call takes its own CUDA stream and staging slot from a pool; at most 16 searches drive the device at once,
//! further callers wait inside the library), so the wrapper is `Send + Sync`.

use std::ffi::CString;
use std::sync::Arc;

use quickwit_search::SearchError;

use crate::ffi;

pub struct GpuContext {
    raw: *mut ffi::QwgpuCtx,
}

// SAFETY: libqwgpu serialises what has to be serialised internally (include/qwgpu.h, "Threading").
unsafe impl Send for GpuContext {}
unsafe impl Sync for GpuContext {}

impl GpuContext {
    /// `device`: CUDA ordinal of the GPU this searcher process owns.
    pub fn new(device: i32) -> Result<Arc<Self>, SearchError> {
        let mut raw = std::ptr::null_mut();
        let rc = unsafe { ffi::qwgpu_init(device, &mut raw) };
        if rc != ffi::QWGPU_OK {
            return Err(ffi::map_error(rc));
        }
        Ok(Arc::new(GpuContext { raw }))
    }

    pub(crate) fn raw(&self) -> *mut ffi::QwgpuCtx {
        self.raw
    }

    /// Cap on the bytes of split data kept in HBM; least recently searched idle splits are evicted beyond it.
    pub fn set_residency_budget(&self, bytes: u64) -> Result<(), SearchError> {
        check(unsafe { ffi::qwgpu_set_residency_budget(self.raw, bytes) })
    }

    /// Largest `max_hits + start_offset` served (1 ..= 20 000; 4096 until set). A root that sends the reference's
    /// limits (10 000 hits from offset up to 10 000) raises it to 20 000.
    pub fn set_max_hits(&self, max_hits: u32) -> Result<(), SearchError> {
        check(unsafe { ffi::qwgpu_set_max_hits(self.raw, max_hits) })
    }

    /// HBM the predicate cache may hold (0, the default, disables it): the doc sets of the queries of paged
    /// (`search_after`) requests, kept per split so that later pages read them. Pass
    /// the capacity of `searcher_config.predicate_cache` (256 MB by default in the reference).
    pub fn set_predicate_cache_budget(&self, bytes: u64) -> Result<(), SearchError> {
        check(unsafe { ffi::qwgpu_set_predicate_cache_budget(self.raw, bytes) })
    }

    /// Makes a split image (include/qwgpu_format.h) resident; the bytes may be dropped afterwards. The counterpart
    /// of `open_split_bundle` + `warmup` (quickwit-search/src/leaf.rs:210-251, 269-472).
    pub fn register_split(&self, split_id: &str, image: &[u8]) -> Result<(), SearchError> {
        let id = CString::new(split_id).map_err(|e| SearchError::InvalidArgument(e.to_string()))?;
        check(unsafe { ffi::qwgpu_split_register(self.raw, id.as_ptr(), image.as_ptr(), image.len() as u64) })
    }

    pub fn unregister_split(&self, split_id: &str) -> Result<(), SearchError> {
        let id = CString::new(split_id).map_err(|e| SearchError::InvalidArgument(e.to_string()))?;
        check(unsafe { ffi::qwgpu_split_unregister(self.raw, id.as_ptr()) })
    }

    pub fn is_resident(&self, split_id: &str) -> bool {
        CString::new(split_id).map(|id| unsafe { ffi::qwgpu_split_is_resident(self.raw, id.as_ptr()) } == 1).unwrap_or(false)
    }

    pub fn resident_bytes(&self) -> u64 {
        unsafe { ffi::qwgpu_resident_bytes(self.raw) }
    }

    /// The predicate cache's budget, bytes held, entries, and hits, misses, fills and evictions so far.
    pub fn predicate_cache_info(&self) -> Result<PredicateCacheInfo, SearchError> {
        let mut i = PredicateCacheInfo::default();
        check(unsafe {
            ffi::qwgpu_predicate_cache_info(self.raw, &mut i.budget_bytes, &mut i.used_bytes, &mut i.entries, &mut i.hits,
                                            &mut i.misses, &mut i.fills, &mut i.evictions)
        })?;
        Ok(i)
    }
}

#[derive(Clone, Copy, Debug, Default)]
pub struct PredicateCacheInfo {
    pub budget_bytes: u64,
    pub used_bytes: u64,
    pub entries: u64,
    pub hits: u64,
    pub misses: u64,
    pub fills: u64,
    pub evictions: u64,
}

impl Drop for GpuContext {
    fn drop(&mut self) {
        unsafe { ffi::qwgpu_shutdown(self.raw) }
    }
}

fn check(rc: i32) -> Result<(), SearchError> {
    if rc == ffi::QWGPU_OK { Ok(()) } else { Err(ffi::map_error(rc)) }
}
