// capi_engine.cpp — C ABI entry points backed by the GPU engine (context, residency, seam C).
#include "engine.h"

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
  r->hits = nullptr;
  r->agg_cells = nullptr;
}

}  // extern "C"
