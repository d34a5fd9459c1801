// capi_core.cpp — error plumbing and trivial entry points of the C ABI (include/qwgpu.h).
#include "common.h"

namespace qw {
static thread_local std::string g_last_error;
void set_last_error(const std::string& msg) { g_last_error = msg; }
}  // namespace qw

extern "C" {
const char* qwgpu_last_error(void) { return qw::g_last_error.c_str(); }
const char* qwgpu_version(void) { return "qwgpu 0.1.0 (sm_90a)"; }
void qwgpu_buf_free(void* buf) { free(buf); }
float qwgpu_bm25_weight(uint64_t doc_freq, uint64_t num_docs, float boost) {
  float w = qw::bm25_idf(doc_freq, num_docs) * (1.0f + qw::BM25_K1);
  return w * boost;
}
float qwgpu_bm25_phrase_weight(const uint64_t* doc_freqs, uint32_t n, uint64_t num_docs, float boost) {
  float idf_sum = 0.0f;  // Bm25Weight::for_terms: the terms' idfs summed in phrase order (f32)
  for (uint32_t i = 0; i < n; i++) idf_sum += qw::bm25_idf(doc_freqs[i], num_docs);
  return idf_sum * (1.0f + qw::BM25_K1) * boost;
}
}
