// capi_engine.cpp — C ABI entry points backed by the GPU engine (context, residency, seam C).
#include "engine.h"
#include "device_types.h"

#define QW_API_BEGIN try {
#define QW_API_END                                   \
  }                                                  \
  catch (const qw::Error& e) {                       \
    qw::set_last_error(e.what());                    \
    return e.code;                                   \
  }                                                  \
  catch (const std::exception& e) {                  \
    qw::set_last_error(e.what());                    \
    return QWGPU_EINTERNAL;                          \
  }

static qw::Engine& engine_of(qwgpu_ctx* ctx) {
  if (!ctx) qw::fail(QWGPU_EINVALID_ARG, "null context");
  if (!ctx->engine) qw::fail(QWGPU_ENODEVICE, "host-only context: no CUDA device bound (there is no CPU search path)");
  return *ctx->engine;
}

extern "C" {

int qwgpu_init(int device, qwgpu_ctx** out) {
  QW_API_BEGIN
  if (!out) qw::fail(QWGPU_EINVALID_ARG, "null out pointer");
  std::unique_ptr<qwgpu_ctx> ctx(new qwgpu_ctx());
  if (device >= 0) ctx->engine.reset(new qw::Engine(device));
  *out = ctx.release();
  return 0;
  QW_API_END
}

void qwgpu_shutdown(qwgpu_ctx* ctx) { delete ctx; }

int qwgpu_split_register(qwgpu_ctx* ctx, const char* split_id, const uint8_t* img, uint64_t img_len) {
  QW_API_BEGIN
  engine_of(ctx).register_split(split_id, img, img_len);
  return 0;
  QW_API_END
}

int qwgpu_split_unregister(qwgpu_ctx* ctx, const char* split_id) {
  QW_API_BEGIN
  engine_of(ctx).unregister_split(split_id);
  return 0;
  QW_API_END
}

int qwgpu_split_register_async(qwgpu_ctx* ctx, const char* split_id, const uint8_t* img, uint64_t img_len) {
  QW_API_BEGIN
  engine_of(ctx).register_split_async(split_id, img, img_len);
  return 0;
  QW_API_END
}

int qwgpu_split_wait(qwgpu_ctx* ctx, const char* split_id) {
  QW_API_BEGIN
  engine_of(ctx).wait_split(split_id);
  return 0;
  QW_API_END
}

int qwgpu_set_residency_budget(qwgpu_ctx* ctx, uint64_t bytes) {
  QW_API_BEGIN
  engine_of(ctx).set_budget(bytes);
  return 0;
  QW_API_END
}

int qwgpu_set_max_hits(qwgpu_ctx* ctx, uint32_t max_hits) {
  QW_API_BEGIN
  if (max_hits < 1 || max_hits > QW_MAX_HITS) qw::fail(QWGPU_EINVALID_ARG, "max_hits limit %u outside [1, 20 000]", max_hits);
  engine_of(ctx).max_hits.store(max_hits, std::memory_order_relaxed);
  return 0;
  QW_API_END
}

int qwgpu_set_predicate_cache_budget(qwgpu_ctx* ctx, uint64_t bytes) {
  QW_API_BEGIN
  engine_of(ctx).set_pred_budget(bytes);
  return 0;
  QW_API_END
}

int qwgpu_predicate_cache_info(qwgpu_ctx* ctx, uint64_t* budget_bytes, uint64_t* used_bytes, uint64_t* entries, uint64_t* hits,
                               uint64_t* misses, uint64_t* fills, uint64_t* evictions) {
  QW_API_BEGIN
  qw::PredCache& c = engine_of(ctx).pred;
  std::lock_guard<std::mutex> g(c.mu);
  uint64_t n = 0;
  for (const auto& s : c.by_split) n += s.second.size();
  if (budget_bytes) *budget_bytes = c.budget;
  if (used_bytes) *used_bytes = c.used.load();
  if (entries) *entries = n;
  if (hits) *hits = c.hits;
  if (misses) *misses = c.misses;
  if (fills) *fills = c.fills;
  if (evictions) *evictions = c.evictions;
  return 0;
  QW_API_END
}

int qwgpu_set_leaf_cache_budget(qwgpu_ctx* ctx, uint64_t bytes) {
  QW_API_BEGIN
  engine_of(ctx).leaf.set_budget(bytes);
  return 0;
  QW_API_END
}

int qwgpu_leaf_cache_info(qwgpu_ctx* ctx, uint64_t* budget_bytes, uint64_t* used_bytes, uint64_t* entries, uint64_t* hits,
                          uint64_t* misses, uint64_t* fills, uint64_t* evictions) {
  QW_API_BEGIN
  qw::LeafCache& c = engine_of(ctx).leaf;
  std::lock_guard<std::mutex> g(c.mu);
  if (budget_bytes) *budget_bytes = c.budget;
  if (used_bytes) *used_bytes = c.used;
  if (entries) *entries = c.lru.size();
  if (hits) *hits = c.hits;
  if (misses) *misses = c.misses;
  if (fills) *fills = c.fills;
  if (evictions) *evictions = c.evictions;
  return 0;
  QW_API_END
}

int qwgpu_residency_info(qwgpu_ctx* ctx, uint64_t* resident_bytes, uint64_t* budget_bytes, uint64_t* num_splits, uint64_t* evictions) {
  QW_API_BEGIN
  qw::Engine& e = engine_of(ctx);
  std::lock_guard<std::mutex> g(e.mu);
  if (resident_bytes) *resident_bytes = e.resident;
  if (budget_bytes) *budget_bytes = e.budget;
  if (num_splits) *num_splits = e.splits.size();
  if (evictions) *evictions = e.evictions;
  return 0;
  QW_API_END
}

int qwgpu_split_is_resident(qwgpu_ctx* ctx, const char* split_id) {
  if (!ctx || !ctx->engine || !split_id) return 0;
  std::lock_guard<std::mutex> g(ctx->engine->mu);
  return ctx->engine->splits.count(split_id) ? 1 : 0;
}

uint64_t qwgpu_resident_bytes(qwgpu_ctx* ctx) {
  if (!ctx || !ctx->engine) return 0;
  std::lock_guard<std::mutex> g(ctx->engine->mu);
  return ctx->engine->resident;
}

int qwgpu_split_search(qwgpu_ctx* ctx, uint32_t num_splits, const char* const* split_ids,
                       const uint8_t* const* plans, const size_t* plan_lens,
                       qwgpu_split_result* results, int* status) {
  QW_API_BEGIN
  qw::Engine& e = engine_of(ctx);
  std::vector<std::shared_ptr<qw::SplitDev>> sp(num_splits);
  std::vector<const uint8_t*> pl(plans, plans + num_splits);
  std::vector<size_t> ln(plan_lens, plan_lens + num_splits);
  for (uint32_t i = 0; i < num_splits; i++) sp[i] = e.find(split_ids[i]);
  std::vector<qw::SplitOutput> outs;
  qw::BatchStats st;
  e.search(sp, pl, ln, outs, st);
  std::string first_err;
  for (uint32_t i = 0; i < num_splits; i++) {
    qwgpu_split_result& r = results[i];
    memset(&r, 0, sizeof r);
    status[i] = outs[i].status;
    if (outs[i].status) { if (first_err.empty()) first_err = outs[i].error; continue; }
    r.num_hits = outs[i].num_hits;
    r.num_partial_hits = (uint32_t)outs[i].hits.size();
    r.num_agg_cells = (uint32_t)outs[i].cells.size();
    if (!outs[i].hits.empty()) {
      r.hits = (QwHit*)malloc(outs[i].hits.size() * sizeof(QwHit));
      memcpy(r.hits, outs[i].hits.data(), outs[i].hits.size() * sizeof(QwHit));
    }
    if (!outs[i].cells.empty()) {
      r.agg_cells = (QwAggCell*)malloc(outs[i].cells.size() * sizeof(QwAggCell));
      memcpy(r.agg_cells, outs[i].cells.data(), outs[i].cells.size() * sizeof(QwAggCell));
    }
    r.num_agg_entries = (uint32_t)outs[i].entries.size();
    if (!outs[i].entries.empty()) {
      r.agg_entries = (QwAggEntry*)malloc(outs[i].entries.size() * sizeof(QwAggEntry));
      memcpy(r.agg_entries, outs[i].entries.data(), outs[i].entries.size() * sizeof(QwAggEntry));
    }
    r.gpu_time_us = st.gpu_time_us;
    r.main_kernel_us = st.main_kernel_us;
    r.num_kernel_launches = st.launches;
    r.exact_fallbacks = st.exact_fallbacks;
    r.postings_scored = outs[i].postings_scored;
    r.algorithmic_bytes = outs[i].algorithmic_bytes;
    r.kernel_mask = st.kernel_mask;
    r.window_docs = st.window_docs;
    r.sample_stride = st.sample_stride;
    r.radix_passes = st.radix_passes;
    r.refined = st.refined;
  }
  if (!first_err.empty()) qw::set_last_error(first_err);
  return 0;
  QW_API_END
}

void qwgpu_split_result_free(qwgpu_split_result* r) {
  if (!r) return;
  free(r->hits);
  free(r->agg_cells);
  free(r->agg_entries);
  r->hits = nullptr;
  r->agg_cells = nullptr;
  r->agg_entries = nullptr;
}

}  // extern "C"
