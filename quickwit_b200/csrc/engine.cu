// engine.cu — host engine: HBM residency of split images, lowering of seam-C plans into the
// window-engine program, batched launches (one launch sequence covers every split of a request),
// top-K threshold selection (sampled fast path + exact radix-select fallback) and result readback.
//
// Replaces, for one leaf request: open_index_with_caches + warmup (quickwit-search/src/leaf.rs:
// 210-251,269-472) at register time, and searcher.search(&query,&collector) (leaf.rs:637) per call.
#include <algorithm>
#include <chrono>
#include <cmath>

#include "ddsketch.h"
#include "engine.h"
#include "kernels.cuh"
#include "union_kernel.cuh"
#include "phrase_kernel.cuh"
#include "termset_kernel.cuh"
#include "driver_kernel.cuh"
#include "agg_kernel.cuh"
#include "trace_kernel.cuh"
#include "composite_kernel.cuh"
#include "deep_select_kernel.cuh"

namespace qw {

#define CUDA_CHECK(expr)                                                                          \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess)                                                                        \
      fail((_e == cudaErrorNoDevice || _e == cudaErrorInsufficientDriver) ? QWGPU_ENODEVICE       \
                                                                           : QWGPU_EINTERNAL,     \
           "CUDA error %s at %s:%d: %s", cudaGetErrorName(_e), __FILE__, __LINE__,               \
           cudaGetErrorString(_e));                                                               \
  } while (0)

uint32_t id_to_fieldnorm(uint8_t id);  // image_builder.cpp

SplitDev::~SplitDev() {
  if (pred) pred->drop_split(this);
  if (d_data) cudaFree(d_data);
  if (d_tabs) cudaFree(d_tabs);
}

// ---- predicate cache (DESIGN.md §4.9) -------------------------------------------------------------
PredEntry::~PredEntry() {
  owner->used.fetch_sub(bytes);
  if (!d_bits) return;
  std::lock_guard<std::mutex> g(owner->free_mu);
  owner->to_free.push_back(d_bits);
}

// Drops the least recently used published entries that no call holds until `limit` bytes or fewer are live (a pinned
// entry stays: a running call reads it). Caller holds `mu`.
bool PredCache::evict_to(uint64_t limit) {
  while (used.load() > limit) {
    std::unordered_map<std::string, std::shared_ptr<PredEntry>>* vm = nullptr;
    std::unordered_map<std::string, std::shared_ptr<PredEntry>>::iterator victim;
    for (auto& s : by_split)
      for (auto e = s.second.begin(); e != s.second.end(); ++e)
        if (e->second.use_count() == 1 && (!vm || e->second->last_use < victim->second->last_use)) { vm = &s.second; victim = e; }
    if (!vm) return false;
    vm->erase(victim);
    evictions++;
  }
  return true;
}

std::shared_ptr<PredEntry> PredCache::acquire(const SplitDev* sp, const std::string& key, uint64_t bytes, bool* hit) {
  std::lock_guard<std::mutex> g(mu);
  auto& m = by_split[sp];
  auto it = m.find(key);
  if (it != m.end()) {
    *hit = true;
    hits++;
    it->second->last_use = ++tick;
    return it->second;
  }
  *hit = false;
  misses++;
  if (bytes > budget || !evict_to(budget - bytes)) return nullptr;
  auto e = std::make_shared<PredEntry>();
  e->owner = this;
  e->key = key;
  e->bytes = bytes;
  e->last_use = ++tick;
  used.fetch_add(bytes);
  return e;
}

void PredCache::publish(const SplitDev* sp, const std::shared_ptr<PredEntry>& e) {
  std::lock_guard<std::mutex> g(mu);
  fills++;
  if (!budget) return;  // (disabled while the call ran: the entry goes)
  e->last_use = ++tick;
  by_split[sp].emplace(e->key, e);  // (a concurrent fill of the same key that published first stays)
}

void PredCache::drop_split(const SplitDev* sp) {
  std::lock_guard<std::mutex> g(mu);
  by_split.erase(sp);
}

void PredCache::free_released(void* stream) {
  std::vector<void*> v;
  {
    std::lock_guard<std::mutex> g(free_mu);
    v.swap(to_free);
  }
  for (void* p : v) cudaFreeAsync(p, (cudaStream_t)stream);
}

// A run's pre-pass records (Run::lay_out): phrases of up to QW_MAX_PHRASE_TERMS terms (k_phrase) and longer ones
// (k_phrase_long), each kernel numbering its driver blocks from 0, the phrases' records outside DPhrase, the term-set
// nodes and their terms. Until Run::stage their addresses are offsets: DPhrase::out into the VBlk region, DPhrase::exp
// into pext, DTermSetNode::bitmap into the bitmap region. A call slot keeps them, so that a call reuses the capacity of
// the calls before it.
struct PrePass {
  std::vector<DPhrase> phr, phl;
  std::vector<DPhraseTerm> pext;
  std::vector<DTermSetNode> tsn;
  std::vector<DTermSetTerm> tst;
  // the batch's instructions whose operand `a` Run::stage sets: an offset into the VBlk or bitmap region, or the device
  // address of a cache entry's bitmap
  struct Operand { uint32_t instr; enum { VBLK, BITMAP, ADDR } kind; uint64_t off; };
  std::vector<Operand> operands;
};

struct CallSlot {
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr, ev3 = nullptr;
  cudaEvent_t ev_block = nullptr;  // cudaEventBlockingSync: waits that yield the CPU (many calls in flight)
  uint8_t *d_blob = nullptr, *h_blob = nullptr;
  size_t blob_cap = 0;
  uint8_t* d_scratch = nullptr;
  size_t scratch_cap = 0;
  uint8_t *d_out = nullptr, *h_out = nullptr;
  size_t out_cap = 0;
  PrePass pre;
  void ensure(size_t blob, size_t scratch, size_t out) {
    if (blob > blob_cap) {
      if (d_blob) cudaFree(d_blob);
      if (h_blob) cudaFreeHost(h_blob);
      blob_cap = blob * 2;
      CUDA_CHECK(cudaMalloc(&d_blob, blob_cap));
      CUDA_CHECK(cudaMallocHost(&h_blob, blob_cap));
    }
    if (scratch > scratch_cap) {
      if (d_scratch) cudaFree(d_scratch);
      scratch_cap = scratch <= ((size_t)1 << 30) ? scratch * 2 : scratch;  // (no headroom for the rare huge call)
      CUDA_CHECK(cudaMalloc(&d_scratch, scratch_cap));
    }
    if (out > out_cap) {
      if (d_out) cudaFree(d_out);
      if (h_out) cudaFreeHost(h_out);
      out_cap = out * 2;
      CUDA_CHECK(cudaMalloc(&d_out, out_cap));
      CUDA_CHECK(cudaMallocHost(&h_out, out_cap));
    }
  }
  ~CallSlot() {
    if (d_blob) cudaFree(d_blob);
    if (h_blob) cudaFreeHost(h_blob);
    if (d_scratch) cudaFree(d_scratch);
    if (d_out) cudaFree(d_out);
    if (h_out) cudaFreeHost(h_out);
    if (ev0) cudaEventDestroy(ev0);
    if (ev_block) cudaEventDestroy(ev_block);
    if (ev1) cudaEventDestroy(ev1);
    if (ev2) cudaEventDestroy(ev2);
    if (ev3) cudaEventDestroy(ev3);
    if (stream) cudaStreamDestroy(stream);
  }
};

// k_trace_replay: the <= 2N-entry map (ordinal + timestamp) and one tile of matched docs in shared memory
static int trace_replay_smem(uint32_t n) { return (int)(12u * (2u * n + QT_TILE)); }

Engine::Engine(int dev) : device(dev) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0)
    fail(QWGPU_ENODEVICE, "no CUDA device available (%s); the qwgpu search path has no CPU fallback",
         e == cudaSuccess ? "0 devices" : cudaGetErrorString(e));
  if (dev >= n) fail(QWGPU_EINVALID_ARG, "device %d out of range (%d devices)", dev, n);
  CUDA_CHECK(cudaSetDevice(dev));
  cudaDeviceProp prop;
  CUDA_CHECK(cudaGetDeviceProperties(&prop, dev));
  sm_count = prop.multiProcessorCount;
  max_smem_optin = (int)prop.sharedMemPerBlockOptin;
  CUDA_CHECK(cudaFuncSetAttribute(qwk::k_window<qwk::MODE_HIST>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem_optin));
  CUDA_CHECK(cudaFuncSetAttribute(qwk::k_window<qwk::MODE_COLLECT>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem_optin));
  CUDA_CHECK(cudaFuncSetAttribute(qwk::k_window<qwk::MODE_COLLECT, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem_optin));
  CUDA_CHECK(cudaFuncSetAttribute(qwk::k_union<qwk::MODE_HIST>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem_optin));
  CUDA_CHECK(cudaFuncSetAttribute(qwk::k_union<qwk::MODE_COLLECT>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem_optin));
  CUDA_CHECK(cudaFuncSetAttribute(qwk::k_union<qwk::MODE_SAMPLE_COLLECT>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem_optin));
  int coop = 0;
  CUDA_CHECK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
  coop_launch = coop != 0;
  CUDA_CHECK(cudaFuncSetAttribute(qwk::k_aggscan, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem_optin));
  CUDA_CHECK(cudaFuncSetAttribute(qwk::k_select, cudaFuncAttributeMaxDynamicSharedMemorySize, 3 * 8 * QW_CAND_CAP));
  CUDA_CHECK(cudaFuncSetAttribute(qwk::k_trace_replay, cudaFuncAttributeMaxDynamicSharedMemorySize, trace_replay_smem(QW_MAX_TOPK)));
}

Engine::~Engine() {
  for (Loader& l : loaders) if (l.t.joinable()) l.t.join();
  cudaSetDevice(device);
  for (CallSlot* s : free_slots) delete s;
  splits.clear();
  pred.by_split.clear();
  pred.free_released(nullptr);
  if (pred.pool) {
    cudaStreamSynchronize(nullptr);
    cudaMemPoolDestroy((cudaMemPool_t)pred.pool);
  }
}

// A budget of 0 disables the cache: every published entry is dropped (the bitmaps of entries a running call still
// holds go when that call releases them). The bitmaps come from a pool of the engine's own that keeps freed memory
// for reuse, so that no search allocates or frees device memory synchronously.
void Engine::set_pred_budget(uint64_t bytes) {
  CUDA_CHECK(cudaSetDevice(device));
  {
    std::lock_guard<std::mutex> g(pred.mu);
    if (bytes && !pred.pool) {
      cudaMemPoolProps props;
      memset(&props, 0, sizeof props);
      props.allocType = cudaMemAllocationTypePinned;
      props.location.type = cudaMemLocationTypeDevice;
      props.location.id = device;
      cudaMemPool_t pool;
      CUDA_CHECK(cudaMemPoolCreate(&pool, &props));
      uint64_t keep = ~0ull;
      CUDA_CHECK(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
      pred.pool = pool;
    }
    pred.budget = bytes;
    if (!bytes) pred.by_split.clear();
    else pred.evict_to(bytes);
  }
  if (!bytes && pred.pool) {
    pred.free_released(nullptr);
    CUDA_CHECK(cudaStreamSynchronize(nullptr));
    CUDA_CHECK(cudaMemPoolTrimTo((cudaMemPool_t)pred.pool, 0));
  }
}

// host half of a registration: directory copy + views (no device work)
static std::shared_ptr<SplitDev> open_split(const char* id, const uint8_t* img, uint64_t len, ImageView* full_out) {
  ImageView full;
  full.open(img, len);
  auto sp = std::make_shared<SplitDev>();
  sp->id = id;
  sp->dir.assign(img, img + full.hdr->data_off);
  // the directory-only view: relax the length check by opening over the original then rebasing
  sp->view = full;
  sp->view.base = sp->dir.data();
  sp->view.hdr = (const QwImgHeader*)sp->dir.data();
  sp->view.fields = (const QwImgField*)(sp->dir.data() + full.hdr->fields_off);
  sp->view.terms = (const QwImgTerm*)(sp->dir.data() + full.hdr->terms_off);
  sp->view.columns = (const QwImgColumn*)(sp->dir.data() + full.hdr->columns_off);
  sp->view.term_bytes = sp->dir.data() + full.hdr->term_bytes_off;
  sp->view.strings = sp->dir.data() + full.hdr->strings_off;
  sp->view.data = nullptr;
  sp->data_len = full.hdr->data_len;
  // bytes columns whose every dictionary entry is a 16-byte trace id (find_trace_ids fails the split otherwise)
  sp->ids16.assign(full.hdr->num_columns, 0);
  for (uint32_t c = 0; c < full.hdr->num_columns; c++) {
    const QwImgColumn& col = sp->view.columns[c];
    if (col.type != QW_COL_BYTES) continue;
    const uint32_t* offs = (const uint32_t*)(sp->view.strings + col.dict_off);
    bool ok = true;
    for (uint32_t k = 0; k < col.dict_num_terms && ok; k++) ok = offs[k + 1] - offs[k] == 16;
    sp->ids16[c] = ok ? 1 : 0;
  }
  *full_out = full;
  return sp;
}

// Bm25Weight cache per field (SURVEY.md Appendix A.3): K1 * (1 - B + B * fieldnorm(id) / avg), followed, per field,
// by the tf-factor table tff[tf][id] = tf / (tf + norm[id]) (tf < 16), built with the same IEEE f32 ops the kernel
// would use, so table lookups are bit-identical to dividing
static std::vector<float> bm25_tables(const ImageView& full) {
  const uint32_t nf = full.hdr->num_fields;
  const size_t kTab = 256 + QW_TFF_ROWS * 256;
  std::vector<float> tabs((size_t)std::max(nf, 1u) * kTab);
  for (uint32_t f = 0; f < nf; f++) {
    // an empty split scores nothing; keep its tables finite
    float avg = full.hdr->num_docs ? (float)full.fields[f].total_num_tokens / (float)full.hdr->num_docs : 1.0f;
    float* t = tabs.data() + f * kTab;
    for (uint32_t i = 0; i < 256; i++)
      t[i] = BM25_K1 * (1.0f - BM25_B + BM25_B * (float)id_to_fieldnorm((uint8_t)i) / avg);
    for (uint32_t tf = 0; tf < QW_TFF_ROWS; tf++)
      for (uint32_t i = 0; i < 256; i++) {
        volatile float num = (float)tf, den = (float)tf + t[i];
        t[256 + tf * 256 + i] = num / den;
      }
  }
  return tabs;
}

// Makes room for `need` more bytes under the budget: drops the least recently searched splits that nothing but
// the table references (a split in use by a running call, or still loading, stays). Caller holds `mu`.
static void evict_for(Engine& e, uint64_t need, const std::string& keep) {
  if (!e.budget) return;
  while (e.resident + need > e.budget) {
    auto victim = e.splits.end();
    for (auto it = e.splits.begin(); it != e.splits.end(); ++it) {
      if (it->first == keep || it->second.use_count() > 1 || it->second->state == 0) continue;
      if (victim == e.splits.end() || it->second->last_use < victim->second->last_use) victim = it;
    }
    if (victim == e.splits.end()) break;  // everything left is in use: over budget until those calls end
    e.resident -= victim->second->data_len;
    e.splits.erase(victim);
    e.evictions++;
  }
}

static void publish(Engine& e, const std::shared_ptr<SplitDev>& sp) {
  auto it = e.splits.find(sp->id);
  if (it != e.splits.end()) e.resident -= it->second->data_len;
  sp->last_use = ++e.tick;
  e.splits[sp->id] = sp;
  e.resident += sp->data_len;
}

void Engine::register_split(const char* id, const uint8_t* img, uint64_t len) {
  ImageView full;
  auto sp = open_split(id, img, len, &full);
  sp->pred = &pred;
  {
    std::lock_guard<std::mutex> g(mu);
    if (budget && sp->data_len > budget) fail(QWGPU_EINVALID_ARG, "split `%s` needs %llu bytes, the residency budget is %llu", id, (unsigned long long)sp->data_len, (unsigned long long)budget);
    evict_for(*this, sp->data_len, sp->id);
  }
  CUDA_CHECK(cudaSetDevice(device));
  CUDA_CHECK(cudaMalloc(&sp->d_data, std::max<uint64_t>(sp->data_len, 16)));
  CUDA_CHECK(cudaMemcpy(sp->d_data, full.data, sp->data_len, cudaMemcpyHostToDevice));
  std::vector<float> tabs = bm25_tables(full);
  CUDA_CHECK(cudaMalloc(&sp->d_tabs, tabs.size() * sizeof(float)));
  CUDA_CHECK(cudaMemcpy(sp->d_tabs, tabs.data(), tabs.size() * sizeof(float), cudaMemcpyHostToDevice));
  std::lock_guard<std::mutex> g(mu);
  publish(*this, sp);
  leaf.drop_split(sp->id);  // (after the publish: a search that reads the cache from here on finds the new image)
}

// Background upload: the split is visible (loading) at once; a loader thread stages the data region through two
// pinned buffers (pageable -> pinned memcpy of chunk i+1 overlaps the DMA of chunk i) on its own stream, so
// searches on other splits keep the GPU while a cold split comes in (leaf.rs:269-472 warmup runs beside searches).
void Engine::register_split_async(const char* id, const uint8_t* img, uint64_t len) {
  ImageView full;
  auto sp = open_split(id, img, len, &full);
  sp->pred = &pred;
  sp->state = 0;
  {
    std::lock_guard<std::mutex> g(mu);
    if (budget && sp->data_len > budget) fail(QWGPU_EINVALID_ARG, "split `%s` needs %llu bytes, the residency budget is %llu", id, (unsigned long long)sp->data_len, (unsigned long long)budget);
    evict_for(*this, sp->data_len, sp->id);
  }
  CUDA_CHECK(cudaSetDevice(device));
  CUDA_CHECK(cudaMalloc(&sp->d_data, std::max<uint64_t>(sp->data_len, 16)));
  std::vector<float> tabs = bm25_tables(full);
  CUDA_CHECK(cudaMalloc(&sp->d_tabs, tabs.size() * sizeof(float)));
  std::lock_guard<std::mutex> g(mu);
  publish(*this, sp);
  leaf.drop_split(sp->id);
  // loaders that have finished (state set, lock released) are reaped here
  for (size_t i = 0; i < loaders.size();) {
    if (loaders[i].sp->state != 0) { loaders[i].t.join(); loaders[i] = std::move(loaders.back()); loaders.pop_back(); }
    else i++;
  }
  loaders.push_back(Loader{std::thread(), sp});
  loaders.back().t = std::thread([this, sp, full, tabs]() {
    std::string err;
    cudaStream_t st = nullptr;
    uint8_t* pin[2] = {nullptr, nullptr};
    cudaEvent_t ev[2] = {nullptr, nullptr};
    const size_t kChunk = 8u << 20;
    auto ok = [&](cudaError_t e, const char* what) { if (e != cudaSuccess && err.empty()) err = std::string(what) + ": " + cudaGetErrorString(e); return e == cudaSuccess; };
    if (ok(cudaSetDevice(device), "cudaSetDevice") && ok(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking), "cudaStreamCreate")) {
      for (int i = 0; i < 2; i++) { ok(cudaMallocHost(&pin[i], kChunk), "cudaMallocHost"); ok(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming), "cudaEventCreate"); }
      uint64_t off = 0;
      for (int k = 0; err.empty() && off < sp->data_len; k ^= 1) {
        const size_t nb = (size_t)std::min<uint64_t>(kChunk, sp->data_len - off);
        ok(cudaEventSynchronize(ev[k]), "upload event");  // the DMA that last used this buffer is done
        memcpy(pin[k], full.data + off, nb);
        ok(cudaMemcpyAsync(sp->d_data + off, pin[k], nb, cudaMemcpyHostToDevice, st), "H2D of the split data");
        ok(cudaEventRecord(ev[k], st), "upload event");
        off += nb;
      }
      ok(cudaMemcpyAsync(sp->d_tabs, tabs.data(), tabs.size() * sizeof(float), cudaMemcpyHostToDevice, st), "H2D of the BM25 tables");
      ok(cudaStreamSynchronize(st), "upload stream");
    }
    for (int i = 0; i < 2; i++) { if (pin[i]) cudaFreeHost(pin[i]); if (ev[i]) cudaEventDestroy(ev[i]); }
    if (st) cudaStreamDestroy(st);
    {
      std::lock_guard<std::mutex> g2(mu);
      sp->load_error = err;
      sp->state = err.empty() ? 1 : 2;
    }
    loaded_cv.notify_all();
  });
}

void Engine::wait_split(const char* id) {
  std::unique_lock<std::mutex> g(mu);
  auto it = splits.find(id);
  if (it == splits.end()) fail(QWGPU_ENOTFOUND, "split '%s' is not registered", id);
  std::shared_ptr<SplitDev> sp = it->second;
  loaded_cv.wait(g, [&] { return sp->state != 0; });
  if (sp->state == 2) fail(QWGPU_EINTERNAL, "upload of split '%s' failed: %s", id, sp->load_error.c_str());
}

void Engine::set_budget(uint64_t bytes) {
  std::lock_guard<std::mutex> g(mu);
  budget = bytes;
  evict_for(*this, 0, "");
}

void Engine::unregister_split(const char* id) {
  std::unique_lock<std::mutex> g(mu);
  auto it = splits.find(id);
  if (it == splits.end()) fail(QWGPU_ENOTFOUND, "split '%s' is not registered", id);
  std::shared_ptr<SplitDev> sp = it->second;
  loaded_cv.wait(g, [&] { return sp->state != 0; });  // (its loader still writes the device buffer)
  it = splits.find(id);
  if (it != splits.end() && it->second == sp) { resident -= sp->data_len; splits.erase(it); }
  sp.reset();  // (the last reference, unless a call still uses the split: its cache entries go with it)
  pred.free_released(nullptr);
  leaf.drop_split(id);
}

// A search takes the split in use: recency for the LRU; a split that is still loading is waited for.
std::shared_ptr<SplitDev> Engine::find(const std::string& id) {
  std::unique_lock<std::mutex> g(mu);
  auto it = splits.find(id);
  if (it == splits.end()) return nullptr;
  std::shared_ptr<SplitDev> sp = it->second;
  loaded_cv.wait(g, [&] { return sp->state != 0; });
  if (sp->state == 2) return nullptr;
  sp->last_use = ++tick;
  return sp;
}

// ---- lowering: QwPlan tree -> window-engine program ----------------------------------------------
struct Lowered {
  DSplitPlan P;
  std::vector<DInstr> instrs;
  std::vector<DCol> cols;
  std::vector<uint64_t> bounds;  // raw-space histogram boundary tables of the fast aggregation path, percentiles
                                 // boundary tables and the sorted raw tables of column sets
  std::vector<uint64_t> col_max_raw;  // parallel to cols: largest bit-packed raw value present in the column
  std::vector<DAgg> aggs;
  std::vector<int> col_map;  // image column -> DCol index
  uint32_t need_cnt = 0, need_ssum = 0, need_msum = 0, levels = 0;  // bit per level
  float score_max = 0.f;
  int fn_field[2] = {-1, -1};
  uint64_t postings = 0, alg_bytes = 0, min_required_df = ~0ull;
  std::vector<std::pair<uint32_t, uint64_t>> range_cols;  // (col, driver df) for roofline accounting
  bool empty = false;                   // a required clause of the root cannot match in this split: no work at all
  // Instructions whose operand `a` is a device address known only once the batch is laid out (Run::lay_out), each
  // with what feeds it: a cache entry's bitmap (entry set), else the VBlk list of phrases[rec] (OP_PHRASE) or the
  // bitmap of the plan's next term-set node (OP_TERM_SET)
  struct Operand { uint32_t instr, rec; std::shared_ptr<PredEntry> entry; };
  std::vector<Operand> operands;
  std::vector<DPhrase> phrases;         // phrase pre-pass records (out / first_work / exp: Run::lay_out)
  std::vector<DPhraseTerm> phrase_ext;  // term records outside DPhrase: the expansions of phrase prefixes and the terms
                                        // of long phrases (phrases[i].exp indexes it)
  std::vector<DTermSetTerm> ts_terms;   // the terms of the term-set nodes, node by node
  uint32_t tr_img_col = 0;              // find_trace_ids: the trace-id column of the image
  uint64_t h_bound = 0;                 // hashed aggregation layout: upper bound on the split's distinct cells
  uint32_t n_agg_cols = 0;              // columns of `cols` first used by an aggregation node (use_col)
  // predicate cache: `pc` is null when every QW_NODE_CACHE is lowered as its child (cache disabled, the plan's
  // stripped lowering, a fill plan)
  PredCache* pc = nullptr;
  bool has_cache = false;                                   // the plan holds a QW_NODE_CACHE
  std::map<uint32_t, std::shared_ptr<PredEntry>> cache_at;  // plan node -> the entry it reads (lower_node's input)
  std::vector<std::shared_ptr<PredEntry>> misses;           // entries this plan fills (published after the call)
  std::shared_ptr<PredEntry> fill;                          // a fill plan: the entry its matches go to
  std::shared_ptr<Lowered> stripped;  // a plan that reads entries: its lowering without the cache (the fallback)
};

// The boundary table of a percentiles node's column (ddsketch.h), built once per split and column: a column that
// spans the whole double range takes a few million logarithms
static std::shared_ptr<const std::vector<uint64_t>> percentiles_table(const SplitDev& sp, uint32_t c) {
  std::lock_guard<std::mutex> g(sp.pct_mu);
  auto it = sp.pct_tables.find(c);
  if (it != sp.pct_tables.end()) return it->second;
  dds::Table t;
  if (!dds::column_table(sp.view.columns[c], true, &t))
    fail(QWGPU_EUNSUPPORTED, "percentiles over a column holding NaN or infinite values are not implemented on the GPU path");
  auto p = std::make_shared<const std::vector<uint64_t>>(std::move(t.edges));
  sp.pct_tables.emplace(c, p);
  return p;
}

// The DCol index of image column c. A column first used by an aggregation node (agg) counts against the aggregations'
// own QW_MAX_AGG_COLS, any other against the QW_MAX_DCOLS of the query and the sort.
static uint32_t use_col(Lowered& L, const SplitDev& sp, uint32_t c, bool agg = false) {
  if (c == 0xFFFFFFFFu) return c;
  if (c >= sp.view.hdr->num_columns) fail(QWGPU_EINVALID_ARG, "plan references column %u (split has %u)", c, sp.view.hdr->num_columns);
  if (L.col_map[c] >= 0) return (uint32_t)L.col_map[c];
  if (agg) {
    if (L.n_agg_cols >= QW_MAX_AGG_COLS)
      fail(QWGPU_EUNSUPPORTED, "aggregations use more than %u columns besides those of the query and sort", QW_MAX_AGG_COLS);
    L.n_agg_cols++;
  } else if (L.cols.size() - L.n_agg_cols >= QW_MAX_DCOLS) fail(QWGPU_EUNSUPPORTED, "plan uses more than %d columns", QW_MAX_DCOLS);
  const QwImgColumn& ic = sp.view.columns[c];
  DCol d;
  d.values_off = ic.values_off; d.index_off = ic.index_off; d.min_value = ic.min_value; d.gcd = ic.gcd;
  d.bits = ic.bits; d.card = ic.cardinality; d.type = ic.type; d.nwords64 = (sp.view.hdr->num_docs + 63) / 64;
  L.col_map[c] = (int)L.cols.size();
  L.cols.push_back(d);
  L.col_max_raw.push_back(ic.gcd ? (ic.max_value - ic.min_value) / ic.gcd : 0);
  return (uint32_t)L.col_map[c];
}

// The cache key of the subtree at `root`: its plan nodes in breadth-first order, children rebased onto that order,
// the root's occur, every boost and bm25_weight zeroed (scores are never read through the cache). On one split these
// nodes fix the doc set exactly. A fill plan's nodes are the key itself.
static std::string pred_key(const QwPlanNode* nodes, uint32_t nn, uint32_t root) {
  std::vector<QwPlanNode> out(1, nodes[root]);
  for (size_t i = 0; i < out.size(); i++) {
    QwPlanNode& n = out[i];
    n.boost = 0.f;
    n.bm25_weight = 0.f;
    const bool parent = n.kind == QW_NODE_BOOL || n.kind == QW_NODE_PHRASE || n.kind == QW_NODE_PHRASE_PREFIX ||
                        n.kind == QW_NODE_TERM_SET || n.kind == QW_NODE_COL_SET || n.kind == QW_NODE_CACHE;
    if (!parent || !n.num_children) { n.first_child = n.num_children = 0; continue; }
    if ((uint64_t)n.first_child + n.num_children > nn || out.size() + n.num_children > nn) fail(QWGPU_EINVALID_ARG, "plan children out of range");
    const uint32_t first = n.first_child, cnt = n.num_children;
    n.first_child = (uint32_t)out.size();
    out.insert(out.end(), nodes + first, nodes + first + cnt);  // (`n` dangles from here)
  }
  out[0].occur = QW_OCCUR_MUST;
  return std::string((const char*)out.data(), out.size() * sizeof(QwPlanNode));
}

// What the node at `idx` is lowered as, when it is a QW_NODE_CACHE: itself when it reads a cache entry (acquired
// here into L.cache_at), else its child (the cache is off for this plan, the node's score is read, or the child is
// ALL / NONE), followed through nested CACHE nodes. Any other node is itself.
static uint32_t resolve_cache(Lowered& L, const SplitDev& sp, const QwPlanNode* nodes, uint32_t nn, uint32_t idx, bool scored) {
  for (uint32_t hops = 0; idx < nn && nodes[idx].kind == QW_NODE_CACHE; hops++) {
    const QwPlanNode& n = nodes[idx];
    if (n.num_children != 1 || n.first_child >= nn || hops >= nn) fail(QWGPU_EINVALID_ARG, "cache node with %u children", n.num_children);
    L.has_cache = true;
    const uint32_t c = n.first_child;
    if (L.pc && !scored && nodes[c].kind != QW_NODE_ALL && nodes[c].kind != QW_NODE_NONE) {
      bool hit = false;
      std::shared_ptr<PredEntry> e = L.pc->acquire(&sp, pred_key(nodes, nn, c), std::max<uint64_t>((sp.view.hdr->num_docs + 31) / 32, 1) * 4, &hit);
      if (e) {
        if (!hit) L.misses.push_back(e);
        L.cache_at[idx] = std::move(e);
        return idx;
      }
    }
    idx = c;
  }
  return idx;
}

// The children of a PHRASE, PHRASE_PREFIX or TERM_SET node `n` (`what` in errors) as terms of this split, all of one
// field. A phrase's field keeps positions and each offset (lo) fits 32 bits; a term set's ords strictly increase.
static std::vector<const QwImgTerm*> term_children(const SplitDev& sp, const QwPlanNode* nodes, const QwPlanNode& n, bool phrase,
                                                   const char* what) {
  std::vector<const QwImgTerm*> terms;
  terms.reserve(n.num_children);
  for (uint32_t i = 0; i < n.num_children; i++) {
    const QwPlanNode& c = nodes[n.first_child + i];
    if (c.kind != QW_NODE_TERM || c.term_ord >= sp.view.hdr->num_terms) fail(QWGPU_EINVALID_ARG, "%s child %u is not a term of this split", what, i);
    const QwImgTerm& t = sp.view.terms[c.term_ord];
    if (i && t.field_id != terms[0]->field_id) fail(QWGPU_EINVALID_ARG, "%s terms of different fields", what);
    if (phrase && !t.pidx_off) fail(QWGPU_EINVALID_ARG, "%s over a field without positions", what);
    if (phrase && c.lo > 0xFFFFFFFFull) fail(QWGPU_EINVALID_ARG, "%s offset out of range", what);
    if (!phrase && i && c.term_ord <= nodes[n.first_child + i - 1].term_ord) fail(QWGPU_EINVALID_ARG, "%s children not in increasing term order", what);
    terms.push_back(&t);
  }
  return terms;
}

static void lower_node(Lowered& L, const SplitDev& sp, const QwPlanNode* nodes, uint32_t nn, uint32_t idx,
                       uint32_t level, uint32_t occur, bool scored_ctx) {
  if (idx >= nn) fail(QWGPU_EINVALID_ARG, "plan node index out of range");
  const QwPlanNode& n = nodes[idx];
  const bool scored = scored_ctx && (occur == QW_OCCUR_MUST || occur == QW_OCCUR_SHOULD);
  DInstr in;
  memset(&in, 0, sizeof in);
  in.level = level;
  in.occur = occur;
  in.flags = scored ? IF_SCORED : 0;
  switch (n.kind) {
    case QW_NODE_TERM: {
      in.op = OP_TERM;
      if (n.term_ord == 0xFFFFFFFFu && level == 0 && (occur == QW_OCCUR_MUST || occur == QW_OCCUR_FILTER)) L.empty = true;
      in.t = L.P.n_terms++;
      if (!qw_program_fits(L.P.n_terms, 0)) fail(QWGPU_EUNSUPPORTED, "more than %d term clauses", QW_MAX_TERMS);
      in.r = 0;
      if (n.term_ord != 0xFFFFFFFFu) {
        if (n.term_ord >= sp.view.hdr->num_terms) fail(QWGPU_EINVALID_ARG, "plan term ord out of range");
        const QwImgTerm& t = sp.view.terms[n.term_ord];
        const QwImgField& f = sp.view.fields[t.field_id];
        in.a = t.data_off; in.b = t.widx_off; in.c = t.skip_off;
        in.n = t.num_blocks; in.m = t.win_shift; in.f = n.bm25_weight;
        in.pad = (uint32_t)((t.sub_off - t.skip_off) >> 4);  // QwSubIdx[] relative to QwSkip[], in 16-byte units
        if (f.flags & QW_FIELD_HAS_FREQS) in.flags |= IF_HAS_TF;
        if (f.flags & QW_FIELD_HAS_FIELDNORMS) in.flags |= IF_HAS_FN;
        L.postings += t.doc_freq;
        L.alg_bytes += t.data_len - t.fn_len - (scored ? 0 : t.tf_len);  // fieldnorm bytes are counted once per plan below
        if (occur == QW_OCCUR_MUST || occur == QW_OCCUR_FILTER) L.min_required_df = std::min<uint64_t>(L.min_required_df, t.doc_freq);
        if (scored) {
          int slot = -1;
          for (int s = 0; s < 2; s++) if (L.fn_field[s] == (int)t.field_id) slot = s;
          if (slot < 0) {
            for (int s = 0; s < 2 && slot < 0; s++) if (L.fn_field[s] < 0) { L.fn_field[s] = (int)t.field_id; slot = s; }
            if (slot < 0) fail(QWGPU_EUNSUPPORTED, "scoring over more than 2 distinct text fields");
          }
          in.r = (uint32_t)slot;
          L.score_max += n.bm25_weight > 0 ? n.bm25_weight : 0.f;
        }
      }
      L.instrs.push_back(in);
      break;
    }
    case QW_NODE_RANGE: case QW_NODE_EXISTS: case QW_NODE_ALL: case QW_NODE_NONE: {
      if (n.kind == QW_NODE_NONE) { in.op = OP_EXISTS; in.r = 0xFFFFFFFFu; }  // matches nothing
      else if (n.kind == QW_NODE_ALL) in.op = OP_ALL;
      else {
        in.op = n.kind == QW_NODE_RANGE ? OP_RANGE : OP_EXISTS;
        in.r = use_col(L, sp, n.column);
        in.a = n.lo; in.b = n.hi;
        if (n.column != 0xFFFFFFFFu) L.range_cols.push_back({n.column, 0});
        // a range that misses the column's [min, max] (the split's own value range) matches nothing
        if (n.kind == QW_NODE_RANGE && n.column != 0xFFFFFFFFu) {
          const QwImgColumn& ic = sp.view.columns[n.column];
          if (ic.num_vals == 0 || n.hi < ic.min_value || n.lo > ic.max_value) in.r = 0xFFFFFFFFu;
        }
      }
      // a required clause at the root that cannot match: the split has no hits (its windows are skipped)
      if (in.r == 0xFFFFFFFFu && in.op != OP_ALL && level == 0 && (occur == QW_OCCUR_MUST || occur == QW_OCCUR_FILTER)) L.empty = true;
      in.f = n.boost;
      if (scored) L.score_max += n.boost > 0 ? n.boost : 0.f;
      L.instrs.push_back(in);
      break;
    }
    case QW_NODE_BOOL: {
      if (level + 1 > QW_MAX_LEVELS) fail(QWGPU_EUNSUPPORTED, "boolean query nested deeper than %d levels", QW_MAX_LEVELS);
      // the bool's own accumulators live at `level`; when it is a child, the caller passed level+1
      DInstr bg;
      memset(&bg, 0, sizeof bg);
      bg.op = OP_BOOL_BEGIN; bg.level = level;
      L.instrs.push_back(bg);
      const size_t first_instr = L.instrs.size();
      L.levels |= 1u << level;
      uint32_t n_req = 0, n_should = 0;
      if (n.first_child + n.num_children > nn) fail(QWGPU_EINVALID_ARG, "plan children out of range");
      // required group: scored MUST clauses in plan order first (fixes the f32 summation order),
      // then unscored required clauses, posting lists before column predicates (so range filters
      // only probe surviving candidates)
      std::vector<uint32_t> order;
      auto child = [&](uint32_t c) -> const QwPlanNode& { return nodes[n.first_child + c]; };
      // what each child is lowered as (resolve_cache), with the child's own occur
      std::vector<uint32_t> eff(n.num_children);
      for (uint32_t c = 0; c < n.num_children; c++)
        eff[c] = resolve_cache(L, sp, nodes, nn, n.first_child + c, scored && (child(c).occur == QW_OCCUR_MUST || child(c).occur == QW_OCCUR_SHOULD));
      auto is_req = [&](uint32_t c) { return child(c).occur == QW_OCCUR_MUST || child(c).occur == QW_OCCUR_FILTER; };
      auto is_colpred = [&](uint32_t c) {
        const uint32_t k = nodes[eff[c]].kind;
        return k == QW_NODE_RANGE || k == QW_NODE_EXISTS || k == QW_NODE_ALL || k == QW_NODE_COL_SET;
      };
      const bool child_scored_ctx = scored_ctx;
      for (uint32_t c = 0; c < n.num_children; c++) if (is_req(c) && child_scored_ctx && child(c).occur == QW_OCCUR_MUST) order.push_back(c);
      for (int pass = 0; pass < 2; pass++)
        for (uint32_t c = 0; c < n.num_children; c++)
          if (is_req(c) && !(child_scored_ctx && child(c).occur == QW_OCCUR_MUST) && (is_colpred(c) ? pass == 1 : pass == 0)) order.push_back(c);
      if (child_scored_ctx) {
        // scored column predicates must also come after posting lists only when that keeps order;
        // scored clauses keep plan order, so nothing to do here
      }
      n_req = (uint32_t)order.size();
      for (uint32_t c = 0; c < n.num_children; c++) if (child(c).occur == QW_OCCUR_SHOULD) { order.push_back(c); n_should++; }
      for (uint32_t c = 0; c < n.num_children; c++) if (child(c).occur == QW_OCCUR_MUST_NOT) order.push_back(c);
      for (uint32_t c : order) {
        const QwPlanNode& cn = child(c);
        uint32_t child_level = nodes[eff[c]].kind == QW_NODE_BOOL ? level + 1 : level;
        if (scored && cn.occur == QW_OCCUR_MUST) L.need_msum |= 1u << level;
        if (scored && cn.occur == QW_OCCUR_SHOULD) L.need_ssum |= 1u << level;
        lower_node(L, sp, nodes, nn, eff[c], child_level, cn.occur, scored);
      }
      uint32_t msm = n.min_should_match == 0xFFFFFFFFu ? 0 : n.min_should_match;
      uint32_t need = msm > 0 ? msm : (n_req == 0 ? 1 : 0);
      if (need >= 2) L.need_cnt |= 1u << level;
      // Scored should-TERMs with a strictly positive weight contribute > 0 to ssum for every matching
      // doc, so their bitmap is (ssum > 0): skip the per-posting bit set and rebuild it at BOOL_END.
      bool any_from_score = false;
      if (need < 2 && scored) {
        for (size_t ii = first_instr; ii < L.instrs.size(); ii++) {
          DInstr& ci = L.instrs[ii];
          if (ci.op == OP_TERM && ci.level == level && ci.occur == QW_OCCUR_SHOULD && (ci.flags & IF_SCORED) && ci.f >= 1e-20f && ci.f < 1e30f) {
            ci.flags |= IF_BITS_FROM_SCORE;
            any_from_score = true;
          }
        }
      }
      DInstr en;
      memset(&en, 0, sizeof en);
      en.op = OP_BOOL_END; en.level = level; en.occur = occur; en.flags = (scored ? IF_SCORED : 0) | (any_from_score ? IF_BITS_FROM_SCORE : 0);
      en.n = n_req; en.m = n_should; en.r = need;
      L.instrs.push_back(en);
      break;
    }
    case QW_NODE_PHRASE: case QW_NODE_PHRASE_PREFIX: {
      // evaluated by a pre-pass (phrase_kernel.cuh) into one uncompressed posting block per block of its driver, the
      // first rarest exact term; the window program consumes those blocks (OP_PHRASE). Up to QW_MAX_PHRASE_TERMS exact
      // terms: k_phrase, the terms inline in DPhrase::t. Longer: k_phrase_long, the terms in phrase_ext, the driver
      // first and then by ascending doc_freq so that candidates die as early as possible (the phrase count is an
      // intersection of position sets: the order cannot change it). A phrase prefix is a phrase of its k exact terms
      // whose last slot is a set of expansions (phrase_ext, k_phrase's suffix stage 2b), never scored.
      const bool prefix = n.kind == QW_NODE_PHRASE_PREFIX;
      if (!prefix && (n.num_children < 2 || n.num_children > QW_MAX_PHRASE_LEN || n.first_child + n.num_children > nn))
        fail(QWGPU_EINVALID_ARG, "phrase node with %u terms", n.num_children);
      const uint32_t k = prefix ? (uint32_t)n.lo : n.num_children;
      if (prefix) {
        if (n.lo < 1 || n.lo >= QW_MAX_PHRASE_TERMS || n.num_children <= k || n.first_child + n.num_children > nn)
          fail(QWGPU_EINVALID_ARG, "phrase prefix node with %llu exact terms and %u children", (unsigned long long)n.lo, n.num_children);
        if (n.num_children - k > QW_MAX_PREFIX_EXPANSIONS)
          fail(QWGPU_EUNSUPPORTED, "phrase prefix with %u expansions (the GPU path takes at most %d)", n.num_children - k, QW_MAX_PREFIX_EXPANSIONS);
        if (scored)
          fail(QWGPU_EUNSUPPORTED, "phrase prefix in a scoring clause of a query ranked by _score is not implemented on the GPU path");
      }
      const std::vector<const QwImgTerm*> terms = term_children(sp, nodes, n, true, prefix ? "phrase prefix" : "phrase");
      for (uint32_t i = k + 1; i < n.num_children; i++)
        if (nodes[n.first_child + i].lo != nodes[n.first_child + k].lo) fail(QWGPU_EINVALID_ARG, "phrase prefix expansions at different offsets");
      // A doc matches when its positions align: term i at c + lo_i for one constant c, which may be negative (tantivy
      // PhraseQuery::new_with_offset after a stop-word filter gives "a@1 b@2"). The kernels take c >= 0, so the offsets
      // are rebased onto the smallest; then c = p - offset for every position p of a term. Refusing a spread of 2^31
      // or more keeps the rebased offsets in 31 bits; positions within one spread of 2^32 compare modulo 2^32.
      uint64_t lo_min = ~0ull, lo_max = 0;
      for (uint32_t i = 0; i < n.num_children; i++) {
        lo_min = std::min<uint64_t>(lo_min, nodes[n.first_child + i].lo);
        lo_max = std::max<uint64_t>(lo_max, nodes[n.first_child + i].lo);
      }
      if (lo_max - lo_min >= (1ull << 31)) fail(QWGPU_EINVALID_ARG, "%s offsets spread over 2^31 positions or more", prefix ? "phrase prefix" : "phrase");
      const uint32_t field_id = terms[0]->field_id;
      const QwImgField& fld = sp.view.fields[field_id];
      const float weight = prefix ? 0.f : n.bm25_weight;
      DPhrase ph;
      memset(&ph, 0, sizeof ph);
      ph.data_base = (uint64_t)sp.d_data;
      ph.n_terms = k;
      ph.n_exp = n.num_children - k;
      ph.weight = weight;
      ph.scored = scored ? 1 : 0;
      ph.fn_off = !prefix && (fld.flags & QW_FIELD_HAS_FIELDNORMS) ? fld.fieldnorm_off : ~0ull;
      if (!prefix) ph.tab = (uint64_t)(sp.d_tabs + (size_t)(256 + QW_TFF_ROWS * 256) * field_id);
      uint64_t best_df = ~0ull;
      for (uint32_t i = 0; i < n.num_children; i++) {
        if (i < k && terms[i]->doc_freq < best_df) { best_df = terms[i]->doc_freq; ph.driver = i; }
        L.alg_bytes += terms[i]->data_len - terms[i]->fn_len;
      }
      const QwImgTerm& drv = *terms[ph.driver];
      auto rec = [&](uint32_t i) {
        const QwImgTerm& t = *terms[i];
        DPhraseTerm pt;
        memset(&pt, 0, sizeof pt);
        pt.data_off = t.data_off; pt.skip_off = t.skip_off; pt.pos_off = t.pos_off; pt.pidx_off = t.pidx_off;
        pt.nblk = t.num_blocks; pt.offset = (uint32_t)(nodes[n.first_child + i].lo - lo_min);
        return pt;
      };
      ph.exp = L.phrase_ext.size();  // the records outside DPhrase: a long phrase's terms, a prefix's expansions
      if (k <= QW_MAX_PHRASE_TERMS) {
        for (uint32_t i = 0; i < k; i++) ph.t[i] = rec(i);
      } else {
        // a stable sort keeps the first rarest term (the driver above) in front
        std::vector<uint32_t> order(k);
        for (uint32_t i = 0; i < k; i++) order[i] = i;
        std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return terms[a]->doc_freq < terms[b]->doc_freq; });
        for (uint32_t i : order) L.phrase_ext.push_back(rec(i));
        ph.driver = 0;
      }
      for (uint32_t i = k; i < n.num_children; i++) L.phrase_ext.push_back(rec(i));
      L.postings += drv.doc_freq;
      L.alg_bytes += (uint64_t)drv.doc_freq * 4 * n.num_children;  // positions probed per candidate (lower bound)
      if (occur == QW_OCCUR_MUST || occur == QW_OCCUR_FILTER) L.min_required_df = std::min<uint64_t>(L.min_required_df, drv.doc_freq);
      in.op = OP_PHRASE;
      in.c = drv.skip_off;
      in.n = drv.num_blocks;
      in.f = weight;
      if (scored) L.score_max += weight > 0 ? weight : 0.f;
      L.operands.push_back({(uint32_t)L.instrs.size(), (uint32_t)L.phrases.size(), nullptr});
      L.phrases.push_back(ph);
      L.instrs.push_back(in);
      break;
    }
    case QW_NODE_TERM_SET: {
      // the pre-pass (termset_kernel.cuh) ORs the children's postings into a doc bitmap; the window program reads it
      // (OP_TERM_SET), never scored
      if (n.num_children < 1 || n.num_children > QW_MAX_SET_TERMS || n.first_child + n.num_children > nn)
        fail(QWGPU_EINVALID_ARG, "term set node with %u terms", n.num_children);
      if (scored)
        fail(QWGPU_EUNSUPPORTED, "term set (regex) in a scoring clause of a query ranked by _score is not implemented on the GPU path");
      // the plan's term-set nodes are numbered in order (every node holds a term)
      const uint32_t node = L.ts_terms.empty() ? 0 : L.ts_terms.back().node + 1;
      uint64_t df = 0;
      for (const QwImgTerm* t : term_children(sp, nodes, n, false, "term set")) {
        DTermSetTerm r;
        memset(&r, 0, sizeof r);
        r.data = (uint64_t)(sp.d_data + t->data_off);
        r.skip = (uint64_t)(sp.d_data + t->skip_off);
        r.nblk = t->num_blocks;
        r.node = node;
        L.ts_terms.push_back(r);
        df += t->doc_freq;
        L.alg_bytes += t->data_len - t->fn_len;
      }
      L.postings += df;
      if (occur == QW_OCCUR_MUST || occur == QW_OCCUR_FILTER) L.min_required_df = std::min<uint64_t>(L.min_required_df, std::min<uint64_t>(df, sp.view.hdr->num_docs));
      in.op = OP_TERM_SET;
      L.operands.push_back({(uint32_t)L.instrs.size(), 0, nullptr});
      L.instrs.push_back(in);
      break;
    }
    case QW_NODE_COL_SET: {
      // a membership test of the column's values (col_match), never scored: the children's values in raw space
      // ((mapped - min) / gcd), sorted, in the call's blob next to the aggregation tables (in.a: an index into L.bounds
      // until the blob is laid out). A value outside the split's [min, max] or off the gcd grid cannot match.
      if (n.num_children < 1 || n.num_children > QW_MAX_SET_TERMS || (uint64_t)n.first_child + n.num_children > nn)
        fail(QWGPU_EINVALID_ARG, "column set node with %u values", n.num_children);
      if (scored)
        fail(QWGPU_EUNSUPPORTED, "column set (term set) in a scoring clause of a query ranked by _score is not implemented on the GPU path");
      for (uint32_t i = 0; i < n.num_children; i++) {
        const QwPlanNode& c = nodes[n.first_child + i];
        if (c.kind != QW_NODE_RANGE || c.column != n.column || c.lo != c.hi)
          fail(QWGPU_EINVALID_ARG, "column set child %u is not a single value of the node's column", i);
        if (i && c.lo <= nodes[n.first_child + i - 1].lo) fail(QWGPU_EINVALID_ARG, "column set children not in increasing value order");
      }
      in.op = OP_COL_SET;
      in.r = use_col(L, sp, n.column);
      in.a = L.bounds.size();
      if (n.column != 0xFFFFFFFFu) {
        L.range_cols.push_back({n.column, 0});
        const QwImgColumn& ic = sp.view.columns[n.column];
        const uint64_t g = ic.gcd ? ic.gcd : 1;
        for (uint32_t i = 0; i < n.num_children && ic.num_vals; i++) {
          const uint64_t v = nodes[n.first_child + i].lo;
          if (v >= ic.min_value && v <= ic.max_value && (v - ic.min_value) % g == 0) L.bounds.push_back((v - ic.min_value) / g);
        }
      }
      in.n = (uint32_t)(L.bounds.size() - in.a);
      if (in.n == 0) in.r = 0xFFFFFFFFu;  // no value can match: like a range that misses the column
      if (in.r == 0xFFFFFFFFu && level == 0 && (occur == QW_OCCUR_MUST || occur == QW_OCCUR_FILTER)) L.empty = true;
      L.instrs.push_back(in);
      break;
    }
    case QW_NODE_CACHE: {
      // a subtree read from its predicate-cache entry (resolve_cache acquired it): the entry's doc bitmap, consumed
      // like a term set's (OP_TERM_SET); a miss is filled by the call's fill pass first
      in.op = OP_TERM_SET;
      L.operands.push_back({(uint32_t)L.instrs.size(), 0, L.cache_at.at(idx)});
      L.instrs.push_back(in);
      break;
    }
    default: fail(QWGPU_EINVALID_ARG, "unknown plan node kind %u", n.kind);
  }
}

static inline uint32_t bits_needed64(uint64_t v) { return v == 0 ? 0 : 64 - __builtin_clzll(v); }

// The aggregation half of lower_plan: the tree's depth and cell layout, one DAgg per node, the find_trace_ids checks,
// then whether the plan takes the fast aggregation path, with its histogram boundary tables
static void lower_aggs(Lowered& L, const SplitDev& sp, const QwPlanHeader* ph, const QwAggNode* aggs) {
  DSplitPlan& P = L.P;
  if (ph->num_aggs > QW_MAX_AGG_NODES) fail(QWGPU_EUNSUPPORTED, "more than %u aggregation nodes", QW_MAX_AGG_NODES);
  for (uint32_t i = 0; i < ph->num_aggs; i++) {
    uint32_t depth = 0;
    for (uint32_t p = aggs[i].parent; p != 0xFFFFFFFFu; p = aggs[p].parent)
      if (p >= ph->num_aggs || ++depth > ph->num_aggs) fail(QWGPU_EINVALID_ARG, "aggregation parent out of range");
    // (the hashed walk keeps one stack frame per level)
    if (depth >= QW_MAX_AGG_LEVELS) fail(QWGPU_EUNSUPPORTED, "aggregations nested more than %u levels deep", QW_MAX_AGG_LEVELS);
  }
  std::vector<uint32_t> bases(ph->num_aggs, 0);
  P.hashed = qw_agg_hashed(aggs, ph->num_aggs) ? 1u : 0u;
  if (P.hashed) L.h_bound = agg_hashed_layout(aggs, ph->num_aggs, sp.view, sp.id.c_str());
  else P.n_cells = (uint32_t)agg_cell_layout(aggs, ph->num_aggs, &bases);
  for (uint32_t i = 0; i < ph->num_aggs; i++) {
    const QwAggNode& a = aggs[i];
    DAgg d;
    memset(&d, 0, sizeof d);
    d.kind = a.kind; d.parent = a.parent; d.first_child = a.first_child; d.num_children = a.num_children;
    d.col = use_col(L, sp, a.column, true); d.num_buckets = a.num_buckets; d.has_bounds = a.has_bounds;
    d.num_ranges = a.num_ranges; d.has_missing = a.has_missing; d.cell_base = bases[i];
    d.interval = a.interval; d.offset = a.offset; d.bound_min = a.bound_min; d.bound_max = a.bound_max;
    d.base_pos = a.base_pos;
    memcpy(d.range_from, a.range_from, sizeof d.range_from);
    memcpy(d.range_to, a.range_to, sizeof d.range_to);
    if ((a.kind == QW_AGG_TERMS || a.kind == QW_AGG_HISTOGRAM) && (a.reserved & QW_AGG_COMP_LEVEL)) {
      d.comp = a.reserved;
      d.comp_after = a.range_from[0];
    }
    if (a.parent != 0xFFFFFFFFu && (aggs[a.parent].kind == QW_AGG_STATS || aggs[a.parent].kind == QW_AGG_PERCENTILES))
      fail(QWGPU_EINVALID_AGG, "metric aggregations cannot have sub-aggregations");
    if (a.kind == QW_AGG_RANGE && a.num_ranges > QW_MAX_AGG_RANGES) fail(QWGPU_EUNSUPPORTED, "more than %d ranges", QW_MAX_AGG_RANGES);
    if (a.kind == QW_AGG_PERCENTILES) {
      // the walk finds a value's bin in the column's boundary table (d.bounds: an index into L.bounds until the blob
      // is laid out); the plan's bin count must be the table's
      std::shared_ptr<const std::vector<uint64_t>> tab;
      if (a.column != 0xFFFFFFFFu) {
        const uint32_t t = sp.view.columns[a.column].type;
        if (t == QW_COL_STR || t == QW_COL_BYTES) fail(QWGPU_EINVALID_AGG, "percentiles over a text or bytes column");
        if (t == QW_COL_IP) fail(QWGPU_EUNSUPPORTED, "percentiles over an ip column are not supported on the GPU path");
        tab = percentiles_table(sp, a.column);
      }
      const uint64_t nb = tab ? tab->size() : 0;
      if (a.num_buckets != nb + (a.has_missing ? 1u : 0u))
        fail(QWGPU_EINVALID_ARG, "percentiles node %u: %u buckets, the split's column has %llu bins", i, a.num_buckets, (unsigned long long)nb);
      d.bounds = L.bounds.size();
      if (tab) L.bounds.insert(L.bounds.end(), tab->begin(), tab->end());
    }
    L.aggs.push_back(d);
  }
  P.n_aggs = ph->num_aggs;
  // (once every node's column and parent are checked: the rule reads the ancestors' columns)
  for (uint32_t i = 0; i < ph->num_aggs; i++)
    if (aggs[i].kind == QW_AGG_STATS) L.aggs[i].is_f64 = qw_stats_sum_exact(sp.view.columns, aggs, i) ? 0u : 1u;
  for (uint32_t i = 0; i < ph->num_aggs; i++) {
    const QwAggNode& a = aggs[i];
    if (a.kind != QW_AGG_TRACE_IDS) continue;
    // FindTraceIdsCollector::for_segment: a missing trace-id bytes column or a timestamp field that is not a date
    // column is an error of the split; an absent timestamp column reads 0 ns for every doc
    if (ph->num_aggs != 1 || ph->max_hits) fail(QWGPU_EINVALID_ARG, "a find_trace_ids node must be the only aggregation of a plan without hits");
    if (a.num_buckets > QW_MAX_TOPK) fail(QWGPU_EUNSUPPORTED, "find_trace_ids with num_traces = %u exceeds the GPU limit %d", a.num_buckets, QW_MAX_TOPK);
    if (a.column >= sp.view.hdr->num_columns || sp.view.columns[a.column].type != QW_COL_BYTES)
      fail(QWGPU_EINTERNAL, "failed to find column for trace_id field");
    if (!sp.ids16[a.column]) fail(QWGPU_EINTERNAL, "the term dictionary of the trace_id field holds a value that is not a 16-byte trace id");
    if (a.reserved != 0xFFFFFFFFu && (a.reserved >= sp.view.hdr->num_columns || sp.view.columns[a.reserved].type != QW_COL_DATETIME))
      fail(QWGPU_EINTERNAL, "the span timestamp field is not a date fast field");
    P.tr_on = 1;
    L.tr_img_col = a.column;
    P.tr_n = a.num_buckets;
    P.tr_num_ords = std::max(sp.view.columns[a.column].dict_num_terms, 1u);
    P.tr_ord_col = L.aggs[i].col;
    P.tr_ts_col = use_col(L, sp, a.reserved, true);
  }
  // fast aggregation path: flat (no nesting) TERMS / HISTOGRAM nodes over always-present single-valued
  // columns; histogram buckets are located through raw-space boundary tables (hist_bounds)
  bool fast = ph->num_aggs > 0 && !P.hashed;
  P.n_stat_cells = 0;
  for (DAgg& d : L.aggs) {
    const bool full_col = d.col != 0xFFFFFFFFu && L.cols[d.col].card == QW_CARD_FULL;
    if (d.kind == QW_AGG_STATS) {
      // stats: top-level, or directly under a top-level bucket node; one {sum, min, max} triple per cell
      if (!full_col || d.num_children || (d.parent != 0xFFFFFFFFu && L.aggs[d.parent].parent != 0xFFFFFFFFu)) fast = false;
      d.stat_base = P.n_stat_cells;
      P.n_stat_cells += d.parent == 0xFFFFFFFFu ? 1u : L.aggs[d.parent].num_buckets;
    } else {
      if (d.parent != 0xFFFFFFFFu || (d.kind != QW_AGG_TERMS && d.kind != QW_AGG_HISTOGRAM) || !full_col ||
          d.num_buckets > QW_SMEM_AGG_CELLS || d.num_buckets == 0)
        fast = false;
    }
  }
  if (!fast) P.n_stat_cells = 0;
  if (fast) {
    for (DAgg& d : L.aggs) {
      if (d.kind != QW_AGG_HISTOGRAM) continue;
      d.bounds = L.bounds.size();  // index for now; turned into a device address when the blob is laid out
      hist_bounds(L.cols[d.col], L.col_max_raw[d.col], d, L.bounds);
      const uint64_t b0 = L.bounds[d.bounds], bn = L.bounds.back();
      d.inv_step = bn > b0 ? (float)((double)d.num_buckets / (double)(bn - b0)) : 0.0f;
    }
  }
  P.fast_aggs = fast ? 1 : 0;
}

static void lower_plan(Lowered& L, const SplitDev& sp, const uint8_t* plan, size_t plan_len, uint32_t max_hits) {
  if (plan_len < sizeof(QwPlanHeader)) fail(QWGPU_EINVALID_ARG, "plan too short");
  const QwPlanHeader* ph = (const QwPlanHeader*)plan;
  if (ph->magic != QW_PLAN_MAGIC) fail(QWGPU_EINVALID_ARG, "bad plan magic");
  size_t need = sizeof(QwPlanHeader) + (size_t)ph->num_nodes * sizeof(QwPlanNode) + (size_t)ph->num_aggs * sizeof(QwAggNode);
  if (plan_len < need || ph->num_nodes == 0) fail(QWGPU_EINVALID_ARG, "plan truncated");
  if (ph->max_hits > max_hits) {
    if (max_hits >= QW_MAX_HITS) fail(QWGPU_EUNSUPPORTED, "max_hits + start_offset = %u exceeds the GPU top-K limit of 20 000", ph->max_hits);
    fail(QWGPU_EUNSUPPORTED, "max_hits + start_offset = %u exceeds the context's GPU top-K limit %u (qwgpu_set_max_hits raises it up to 20 000)",
         ph->max_hits, max_hits);
  }
  const QwPlanNode* nodes = (const QwPlanNode*)(plan + sizeof(QwPlanHeader));
  const QwAggNode* aggs = (const QwAggNode*)(nodes + ph->num_nodes);
  memset(&L.P, 0, sizeof L.P);
  L.col_map.assign(sp.view.hdr->num_columns, -1);
  DSplitPlan& P = L.P;
  P.data_base = (uint64_t)sp.d_data;
  P.num_docs = sp.view.hdr->num_docs;
  P.max_hits = ph->max_hits;
  P.scoring = ph->scoring;
  P.sa = ph->search_after;
  P.score_hits = (uint32_t)qw_plan_score_hits(ph);
  const bool scoring = ph->scoring != 0;
  const uint32_t root = resolve_cache(L, sp, nodes, ph->num_nodes, 0, scoring);
  if (nodes[root].kind == QW_NODE_BOOL) {
    lower_node(L, sp, nodes, ph->num_nodes, root, 0, QW_OCCUR_MUST, scoring);
  } else if (nodes[root].kind == QW_NODE_TERM && scoring) {
    // a scored single-term query is the one-clause case of the BM25 union: lower it as
    // bool{should: [term]} so that it takes k_union (same matches, same f32 score)
    QwPlanNode wrap[2];
    memset(wrap, 0, sizeof wrap);
    wrap[0].kind = QW_NODE_BOOL; wrap[0].occur = QW_OCCUR_MUST; wrap[0].boost = 1.0f;
    wrap[0].first_child = 1; wrap[0].num_children = 1; wrap[0].min_should_match = 0xFFFFFFFFu;
    wrap[1] = nodes[root];
    wrap[1].occur = QW_OCCUR_SHOULD;
    lower_node(L, sp, wrap, 2, 0, 0, QW_OCCUR_MUST, scoring);
  } else {
    DInstr bg; memset(&bg, 0, sizeof bg); bg.op = OP_BOOL_BEGIN; L.instrs.push_back(bg);
    L.levels |= 1;
    if (scoring) L.need_msum |= 1;
    lower_node(L, sp, nodes, ph->num_nodes, root, 0, QW_OCCUR_MUST, scoring);
    DInstr en; memset(&en, 0, sizeof en); en.op = OP_BOOL_END; en.n = 1; en.flags = scoring ? IF_SCORED : 0; L.instrs.push_back(en);
  }
  {
    // root bool == pure OR of positive-weight scored terms (the BM25 top-K shape): the collect pass can
    // take matches, hit count and the next window's zeroed accumulator straight from the score array
    const DInstr& last = L.instrs.back();
    bool pure = last.op == OP_BOOL_END && last.level == 0 && (last.flags & IF_BITS_FROM_SCORE) && last.n == 0 && last.r == 1;
    for (const DInstr& in : L.instrs) {
      if (in.op == OP_BOOL_BEGIN || in.op == OP_BOOL_END) { if (in.level != 0) pure = false; continue; }
      if (!(in.op == OP_TERM && in.occur == QW_OCCUR_SHOULD && (in.flags & IF_BITS_FROM_SCORE))) pure = false;
    }
    L.P.fused_score_root = pure ? 1 : 0;
  }
  if (!qw_program_fits(L.P.n_terms, L.instrs.size())) fail(QWGPU_EUNSUPPORTED, "query too large for the GPU program (%zu > %d instructions)", L.instrs.size(), QW_MAX_INSTR);
  P.n_instr = (uint32_t)L.instrs.size();
  uint32_t nl = 0;
  while (L.levels >> nl) nl++;
  P.n_levels = nl;
  // fieldnorm / BM25 slots
  for (int s = 0; s < 2; s++) {
    P.fn_off[s] = ~0ull;
    if (L.fn_field[s] >= 0) {
      const QwImgField& f = sp.view.fields[L.fn_field[s]];
      P.n_fn_slots = s + 1;
      P.bm25_tab[s] = (uint64_t)(sp.d_tabs + (size_t)(256 + QW_TFF_ROWS * 256) * L.fn_field[s]);
      if (f.flags & QW_FIELD_HAS_FIELDNORMS) {
        P.fn_off[s] = f.fieldnorm_off;
        L.alg_bytes += std::min<uint64_t>(L.postings, P.num_docs);
      }
    }
  }
  // sort / key spec (sort_by_from_request, quickwit-search/src/collector.rs:994-1030)
  DKeySpec& ks = P.key;
  for (int i = 0; i < 2; i++) {
    ks.kind[i] = ph->sort[i].kind; ks.order[i] = ph->sort[i].order; ks.col[i] = 0xFFFFFFFFu;
    if (ph->sort[i].kind == QW_SORT_COLUMN) {
      if (ph->sort[i].column == 0xFFFFFFFFu) ks.kind[i] = i == 0 ? (uint32_t)QW_SORT_DOCID : (uint32_t)QW_SORT_NONE;  // all None
      else {
        uint32_t t = sp.view.columns[ph->sort[i].column].type;
        if (t == QW_COL_STR) fail(QWGPU_EINVALID_ARG, "Unsupported sort field type `Str`.");
        if (t == QW_COL_IP) fail(QWGPU_EINVALID_ARG, "Unsupported sort field type `IpAddr`.");
        ks.col[i] = use_col(L, sp, ph->sort[i].column);
      }
    }
  }
  if (ks.kind[1] == QW_SORT_DOCID) ks.kind[1] = QW_SORT_NONE;  // _doc as 2nd key extracts None
  if (ks.kind[0] == QW_SORT_NONE) ks.kind[0] = QW_SORT_DOCID;
  if (ks.kind[1] == QW_SORT_NONE) ks.order[1] = QW_ORDER_DESC;  // SortByPair::sort_orders default
  ks.score_scale = 0.f;
  ks.doc_bits = bits_needed64(P.num_docs ? P.num_docs - 1 : 0);
  ks.total_bits = ks.doc_bits;
  for (int i = 0; i < 2; i++) {
    ks.rbits[i] = 0; ks.hasbit[i] = 0; ks.raw_max[i] = 0;
    if (ks.kind[i] == QW_SORT_SCORE) {
      ks.hasbit[i] = 1;
      ks.rbits[i] = i == 0 ? 42 : 32;  // [lin:10 |] order-preserving f32 bits
    } else if (ks.kind[i] == QW_SORT_COLUMN) {
      const uint32_t bits = L.cols[ks.col[i]].bits;
      ks.hasbit[i] = 1;
      ks.rbits[i] = bits;
      ks.raw_max[i] = bits == 64 ? ~0ull : ((1ull << bits) - 1);
    }
    ks.total_bits += ks.hasbit[i] + ks.rbits[i];
  }
  ks.narrow = ks.total_bits <= 64 ? 1 : 0;
  {
    uint32_t pos = 0;
    for (int i = 0; i < 2; i++) {
      ks.sh_has[i] = ks.hasbit[i] ? 64 - pos - 1 : 0;
      pos += ks.hasbit[i];
      ks.sh_r[i] = (ks.narrow && ks.rbits[i]) ? 64 - pos - ks.rbits[i] : 0;
      pos += ks.rbits[i];
    }
    ks.sh_doc = (ks.narrow && ks.doc_bits) ? 64 - pos - ks.doc_bits : 0;
    if (!ks.narrow) ks.sh_has[0] = ks.sh_has[1] = 0;
  }
  if (ks.kind[0] == QW_SORT_SCORE) {
    float smax = L.score_max > 1e-30f ? L.score_max : 1.0f;
    ks.score_scale = 1024.0f / smax;
    ks.top_mode = QW_TOP_SCORE;
  } else if (ks.kind[0] == QW_SORT_COLUMN && ks.rbits[0] >= 10) ks.top_mode = QW_TOP_COLUMN;
  else if (ks.kind[0] == QW_SORT_DOCID && ks.kind[1] == QW_SORT_NONE && ks.doc_bits >= 11) ks.top_mode = QW_TOP_DOC;
  else ks.top_mode = QW_TOP_FULL;
  lower_aggs(L, sp, ph, aggs);
  P.n_cols = (uint32_t)L.cols.size();
}

// Consecutive regions of one buffer or shared-memory block: each starts where the one before ends, rounded up to
// `align` bytes
struct Arena {
  size_t align, off = 0;
  size_t take(size_t bytes) { const size_t o = off; off = (off + bytes + align - 1) & ~(align - 1); return o; }
};

// shared-memory arena for a batch (max over the batch's plans)
static uint32_t stage_bytes_for(uint32_t W) {
  return std::min<uint32_t>(std::max<uint32_t>(W, 8192), 24576);
}

static SmemLayout make_layout(uint32_t W, uint32_t n_levels, uint32_t need_cnt, uint32_t need_msum, uint32_t need_ssum,
                              uint32_t max_instr, uint32_t max_cols, uint32_t max_aggs, uint32_t n_fn, bool rec_l0, bool rangeq) {
  SmemLayout L;
  memset(&L, 0xFF, sizeof L);
  Arena a{16};
  L.misc = a.take(32 + 4 * QW_MAX_TERMS + QW_MAX_TERMS);  // counters, per-term block bases, per-term instruction index
  L.instr = a.take(std::max(max_instr, 1u) * sizeof(DInstr));
  L.cols = a.take(std::max(max_cols, 1u) * sizeof(DCol));
  L.aggs = a.take(std::max(max_aggs, 1u) * sizeof(DAgg));
  L.key = a.take(sizeof(DKeySpec));

  for (uint32_t l = 0; l < n_levels; l++) {
    L.lvl[l].req = a.take(W / 8);
    L.lvl[l].shd = a.take(W / 8);
    L.lvl[l].nt = a.take(W / 8);
    if ((need_cnt >> l) & 1) L.lvl[l].cnt = a.take(W);
    if ((need_msum >> l) & 1) L.lvl[l].msum = a.take(W * 4);
    if ((need_ssum >> l) & 1) L.lvl[l].ssum = a.take(W * 4);
    L.lvl[l].rsc = L.lvl[l].msum != 0xFFFFFFFFu ? L.lvl[l].msum : L.lvl[l].ssum;
  }
  L.tmp = a.take(W / 8);
  for (uint32_t s = 0; s < n_fn; s++) L.fn[s] = a.take(W);  // BM25 tables stay in global memory (L1-resident)
  L.rng = a.take(QW_MAX_TERMS * 16);
  L.hitq = L.rng;  // the collect-time hit queues alias rng / blkrec / termblk (contiguous, dead after the program)
  L.blkrec = a.take(QW_MAX_WBLK * 8);
  L.termblk = a.take(QW_MAX_TERMS * 8);
  L.stage = a.take(stage_bytes_for(W));
  L.hist = L.stage;  // histogram / privatised aggregation counters reuse the staging area at collect time
  if (rec_l0) L.l0hist = a.take(QW_HIST_BINS * 4);
  if (rangeq) L.rangeq = a.take(QW_WARPS * (32 + 32 * 4) * 2);  // QW_WARPS x QW_HITQ_CAP uint16 (kernels.cuh)
  L.total = a.off;
  return L;
}

// shared-memory arena of the BM25-union pipeline (union_kernel.cuh): score array, QU_SLOTS staging slots
// (block payload + records + per-term table + header), mbarriers, MODE_HIST histogram, MODE_SAMPLE_COLLECT thresholds
// (its sample histogram takes a held slot's payload)
static qwk::USmem make_union_layout(uint32_t W, bool hist, bool sample, uint32_t budget) {
  qwk::USmem L;
  memset(&L, 0, sizeof L);
  Arena a{16};
  L.score = a.take(W * 4);
  L.bars = a.take(8 * (2 * QU_SLOTS + QU_CHAIN));
  if (hist) L.hist = a.take(QW_HIST_BINS * 4);
  L.cands = a.take(QU_NCW * QU_CANDS * 8 + QU_NCW * 4);
  if (sample) L.thr = a.take(2 * sizeof(DThresh) + 2 * 4 + 2 * 4);
  const uint32_t off = (uint32_t)a.off, fixed = QU_MAXBLK * 16 + QU_MAX_TERMS * 16 + 32 + QU_PAD;
  const uint32_t cap = budget > off + QU_SLOTS * (fixed + 2048) ? ((budget - off) / QU_SLOTS - fixed) & ~15u : 2048;
  L.cap = cap;
  L.payload = 0;
  L.recs = cap + QU_PAD;
  L.ttab = L.recs + QU_MAXBLK * 16;
  L.hdr = L.ttab + QU_MAX_TERMS * 16;
  L.slot_stride = L.hdr + 48;  // header (32 B) + block hand-out counter
  L.slot0 = a.take(QU_SLOTS * L.slot_stride);
  L.total = a.off;
  return L;
}

// the BM25 top-K shape, [BOOL_BEGIN, TERM x n, BOOL_END] ranked by _score: the BM25-union pipeline (k_union)
static bool union_eligible(const Lowered& L) {
  return L.P.fused_score_root && L.P.max_hits && !L.P.sa.present && !L.P.n_aggs && L.P.key.kind[0] == QW_SORT_SCORE &&
         L.P.key.order[0] == QW_ORDER_DESC && L.P.n_terms <= QU_MAX_TERMS && L.P.n_instr == L.P.n_terms + 2;
}

// one driving posting list + required column filters, no aggregations: the posting-driven kernel
// (driver_kernel.cuh). [BOOL_BEGIN, TERM, (RANGE | EXISTS | COL_SET) x 0..4, BOOL_END] at level 0.
static bool driver_eligible(const Lowered& L) {
  const std::vector<DInstr>& I = L.instrs;
  if (!(L.P.n_aggs == 0 && I.size() >= 3 && I.size() <= 3 + QD_MAX_FILTERS && I[0].op == OP_BOOL_BEGIN && I[1].op == OP_TERM &&
        I.back().op == OP_BOOL_END && I.back().level == 0))
    return false;
  const bool req = I[1].occur == QW_OCCUR_MUST || I[1].occur == QW_OCCUR_FILTER;
  if (!req && !(I[1].occur == QW_OCCUR_SHOULD && I.size() == 3 && I.back().r == 1 && I.back().n == 0)) return false;
  for (size_t k = 2; k + 1 < I.size(); k++) {
    const bool colpred = I[k].op == OP_RANGE || I[k].op == OP_EXISTS || I[k].op == OP_COL_SET;
    const bool unscored_req = I[k].occur == QW_OCCUR_FILTER || (I[k].occur == QW_OCCUR_MUST && !(I[k].flags & IF_SCORED));
    if (!colpred || !unscored_req || I[k].level != 0) return false;
  }
  return true;
}

// match_all + 1..QA_MAX_AGGS flat terms / histogram aggregations, no hits: the streaming column kernel (agg_kernel.cuh).
// Lays out its shared memory; false when a plan does not qualify or the layout does not fit (wider plans run on
// k_window).
static bool aggscan_layout(const std::vector<Lowered>& low, int max_smem_optin, qwk::ASmem* alay) {
  uint32_t maxbits[QA_MAX_AGGS] = {0}, a_cells = 1;
  for (const Lowered& L : low) {
    if (!(L.P.n_instr == 3 && L.instrs[1].op == OP_ALL && L.P.max_hits == 0 && L.P.n_aggs > 0 && L.P.n_aggs <= QA_MAX_AGGS &&
          L.P.n_cells <= QA_MAX_CELLS))
      return false;
    for (uint32_t gi = 0; gi < L.P.n_aggs; gi++) {
      const DAgg& d = L.aggs[gi];
      const bool flat = d.parent == 0xFFFFFFFFu && d.num_children == 0 && (d.kind == QW_AGG_TERMS || d.kind == QW_AGG_HISTOGRAM) && !d.has_missing;
      if (!flat || !L.P.fast_aggs || d.col == 0xFFFFFFFFu || L.cols[d.col].card != QW_CARD_FULL || L.cols[d.col].bits > 32) return false;
      maxbits[gi] = std::max(maxbits[gi], L.cols[d.col].bits);
    }
    a_cells = std::max(a_cells, L.P.n_cells);
  }
  memset(alay, 0, sizeof *alay);
  Arena slot{16};
  for (uint32_t gi = 0; gi < QA_MAX_AGGS; gi++) alay->col_off[gi] = slot.take(maxbits[gi] ? QA_CHUNK / 8 * maxbits[gi] + 16 : 0);
  alay->hdr = slot.take(16);
  alay->slot_stride = slot.off;
  Arena a{16};
  alay->bars = a.take(8 * 2 * QA_SLOTS);
  alay->atab = a.take(QA_MAX_AGGS * sizeof(qwk::AggRow));
  alay->bcache = a.take(QA_CW * QA_MAX_AGGS * 16);
  alay->cells = a.take(a_cells * 4);
  alay->slot0 = a.take(QA_SLOTS * alay->slot_stride);
  alay->total = a.off;
  return (int)alay->total + 1024 <= max_smem_optin;
}

// The kernel route of a batch and everything it fixes: window sizes, the threshold sample, the work lists and the
// shared-memory layouts. A pass that the route's own kernel does not serve runs on k_window with `lay`.
struct Route {
  enum Kind { WINDOW, DRIVER, UNION, AGGSCAN } kind = WINDOW;
  uint32_t W = 0, W_h = 0;   // docs per window: collect and exact radix passes / sampled threshold pass
  uint32_t stride = 1;       // threshold sample: every stride-th window (driver: posting block)
  bool edge_sample = false;  // the sample is the explicit list `sample_win`: strided windows + each split's first and last
  bool rec_l0 = false;       // the collect pass records the exact level-0 histogram (second-chance top-K)
  SmemLayout lay;             // k_window
  qwk::USmem ulay_c, ulay_h, ulay_s;  // k_union collect / histogram / collect with its own sample
  qwk::ASmem alay;            // k_aggscan
  // prefix sums over splits: windows, sampled windows; driver: posting blocks, sampled blocks ([n + 1] or empty)
  std::vector<uint32_t> fw_all, fw_smp, fw_drv, fw_dsm, sample_win;  // sample_win: window | edge << 31 per work item
  // k_driver runs every pass without refine flags, at any radix level; k_union the collect pass and the level-0
  // histogram without a prefix; k_aggscan the plain collect pass
  bool serves(int mode, uint32_t level, uint32_t use_prefix, uint32_t flags) const {
    return !flags && (kind == DRIVER || (kind == UNION && (mode == qwk::MODE_COLLECT || (level == 0 && !use_prefix))) ||
                      (kind == AGGSCAN && mode == qwk::MODE_COLLECT));
  }
};

// the threshold sample and the work lists of the route's window size
static void plan_sample(Route& r, const std::vector<Lowered>& low, int sm_count) {
  const uint32_t n = (uint32_t)low.size();
  auto windows = [](const Lowered& L, uint32_t W) { return L.empty ? 0u : (L.P.num_docs + W - 1) / W; };
  // BM25-union batches sample the threshold over the collect pass's window size rounded down to 1024 docs. Finer
  // windows (the same fraction of the docs in more work items) were measured on the bench workload, one H100 80GB HBM3
  // (400 W power limit): W gives 1.175-1.183 ms per 4-query step, W / 2 gives 1.194-1.203 ms and W / 4 gives
  // 1.216-1.231 ms (the per-window clause chain does not shrink with the window).
  r.W_h = r.kind == Route::UNION ? std::max(1024u, r.W & ~1023u) : r.W;
  uint32_t mw = 0, tw = 0;
  for (const Lowered& L : low) { mw = std::max(mw, windows(L, r.W_h)); tw += windows(L, r.W_h); }
  // sampling stride of the threshold-estimation pass: 1/16 of the windows (a coarser sample shortens the histogram
  // pass, but the looser threshold lets more candidates through the collect pass)
  const uint32_t stride_cap = 16;
  r.stride = std::min(stride_cap, std::max(1u, mw / 8));
  if (r.kind == Route::UNION) {
    // Large requests: at most ONE sampled window per resident block (the sampled pass is latency bound — a block
    // that gets two windows doubles its duration), up to a stride of 32. Bench workload on one H100 80GB HBM3 (400 W
    // power limit; 6528 windows, 132 SMs x 2 = 264 blocks): stride 25 instead of 16, 1.175-1.183 against 1.209-1.211 ms
    // per 4-query step (a fixed stride of 32: 1.174-1.181 ms, no better).
    const uint32_t per_block = (tw + (uint32_t)(sm_count * QU_MINB) - 1) / (uint32_t)(sm_count * QU_MINB);
    r.stride = std::max(r.stride, std::min({per_block, 32u, std::max(1u, mw / 8)}));
  }
  if (r.kind == Route::DRIVER) {
    // posting-driven kernel: the work list is the driving term's posting blocks; the threshold sample takes every
    // stride-th BLOCK (128 postings, fine enough for keys that follow doc order: what lies between two sampled
    // blocks is < 2K postings)
    uint32_t max_blocks = 0;
    for (const Lowered& L : low) max_blocks = std::max(max_blocks, L.empty ? 0u : L.instrs[1].n);
    r.stride = std::min(stride_cap, std::max(1u, max_blocks / 64));
    r.fw_drv.assign(n + 1, 0);
    r.fw_dsm.assign(n + 1, 0);
    for (uint32_t i = 0; i < n; i++) {
      const uint32_t nb = low[i].empty ? 0u : low[i].instrs[1].n;
      r.fw_drv[i + 1] = r.fw_drv[i] + nb;
      r.fw_dsm[i + 1] = r.fw_dsm[i] + qw_sample_count(nb, i, r.stride);
    }
  }
  // the generic kernels sample an explicit window list: strided windows + the first and last window of each
  // split (weight 1 in the histogram); the union pipeline keeps the plain strided sample (scores do not
  // follow doc order)
  r.edge_sample = r.kind != Route::UNION && r.kind != Route::DRIVER && r.stride > 1;
  r.fw_all.assign(n + 1, 0);
  r.fw_smp.assign(n + 1, 0);
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t nw = windows(low[i], r.W_h);
    r.fw_all[i + 1] = r.fw_all[i] + windows(low[i], r.W);
    if (r.edge_sample) {  // (stride > 1)
      uint32_t cnt = 0;
      for (uint32_t w = 0; w < nw; w++) {
        const bool edge = w == 0 || w + 1 == nw, strided = w % r.stride == i % r.stride;
        if (edge || strided) { r.sample_win.push_back(w | (edge ? 0x80000000u : 0u)); cnt++; }
      }
      r.fw_smp[i + 1] = r.fw_smp[i] + cnt;
    } else r.fw_smp[i + 1] = r.fw_smp[i] + qw_sample_count(nw, i, r.stride);
  }
}

// fill: a predicate-cache fill batch, which only k_window serves (it writes the match words out)
static Route choose_route(const std::vector<Lowered>& low, int max_smem_optin, int sm_count, bool fill = false) {
  Route r;
  uint32_t n_levels = 1, need_cnt = 0, need_ssum = 0, need_msum = 0, max_instr = 0, max_cols = 0, max_aggs = 0, n_fn = 0;
  // second-chance top-K: when no plan ranks by _score first, the collect pass also records the exact
  // level-0 histogram and every window's best digit, so that a failed sampled threshold is repaired
  // by a candidates-only pass over the few windows that can hold candidates
  bool rec_l0 = true, rangeq = false, any_topk = false, all_union = true, all_driver = true;
  for (const Lowered& L : low) {
    all_union = all_union && union_eligible(L);
    all_driver = all_driver && driver_eligible(L);
    if (L.P.max_hits && L.P.key.kind[0] == QW_SORT_SCORE) rec_l0 = false;
    for (const DInstr& in : L.instrs)
      if ((in.op == OP_RANGE || in.op == OP_EXISTS || in.op == OP_COL_SET) && (in.occur == QW_OCCUR_MUST || in.occur == QW_OCCUR_FILTER)) rangeq = true;
    n_levels = std::max(n_levels, L.P.n_levels);
    need_cnt |= L.need_cnt; need_ssum |= L.need_ssum; need_msum |= L.need_msum;
    max_instr = std::max(max_instr, L.P.n_instr); max_cols = std::max(max_cols, L.P.n_cols); max_aggs = std::max(max_aggs, L.P.n_aggs);
    n_fn = std::max(n_fn, L.P.n_fn_slots);
    any_topk |= L.P.max_hits > 0;
  }
  if (fill) r.kind = Route::WINDOW;
  else if (all_driver) r.kind = Route::DRIVER;
  else if (all_union) r.kind = Route::UNION;
  else if (aggscan_layout(low, max_smem_optin, &r.alay)) r.kind = Route::AGGSCAN;
  r.rec_l0 = rec_l0 && any_topk && r.kind != Route::DRIVER;
  // (union batches: k_window is only the rare exact-radix fallback)
  const int smem_per_block = max_smem_optin / (r.kind == Route::UNION ? 1 : QW_MIN_BLOCKS_PER_SM);
  auto layout = [&](uint32_t W) {
    return make_layout(W, n_levels, need_cnt, need_msum, need_ssum, max_instr, max_cols, max_aggs, n_fn, r.rec_l0, rangeq);
  };
  // k_aggscan's flat work list is the list of QA_CHUNK-doc chunks: the generic layout must take a whole chunk
  if (r.kind == Route::AGGSCAN && (int)layout(QA_CHUNK).total + 1024 > smem_per_block) r.kind = Route::WINDOW;
  // window size: as large as shared memory allows for the configured blocks/SM (per-window fixed
  // costs — staging, program interpretation, barriers — amortise over more postings). BM25-union batches run the
  // TMA + mbarrier pipeline (union_kernel.cuh): fixed 15360-doc windows, two blocks per SM
  r.W = r.kind == Route::AGGSCAN ? QA_CHUNK : r.kind == Route::UNION ? 15360u * 2 / QU_MINB : 32768u;
  for (;; r.W >>= 1) {
    r.lay = layout(r.W);
    if ((int)r.lay.total + 1024 <= smem_per_block || r.W == 1024) break;
  }
  if ((int)r.lay.total > max_smem_optin) fail(QWGPU_EUNSUPPORTED, "query needs %u bytes of shared memory per block", r.lay.total);
  if (r.kind == Route::UNION) {
    // (the generic layout above stays valid for the same W: exact radix passes below level 0 use k_window)
    const uint32_t u_budget = (uint32_t)(max_smem_optin + 1024) / QU_MINB - 1024 - 64;
    r.ulay_c = make_union_layout(r.W, false, false, u_budget);
    r.ulay_h = make_union_layout(r.W, true, false, u_budget);
    r.ulay_s = make_union_layout(r.W, false, true, u_budget);
  }
  plan_sample(r, low, sm_count);
  return r;
}

// A call slot from the pool, behind the admission gate; both are given back when the call ends, on every path.
// Admission: at most QWGPU_MAX_IN_FLIGHT (default 16) searches drive the device at once; further callers wait here
// on a condition variable (no CUDA calls, no spinning). Measured on the mixed config-5 query set from 64 host threads,
// one H100 80GB HBM3 (400 W power limit): with the limit at 16, 1643 queries/s (p99 66-72 ms) in both of two runs;
// with it at 64, 894 and 1517 queries/s (p99 341 and 174 ms) — the driver's per-context lock and 64 interleaved
// streams cost more than the extra overlap brings.
struct SlotLease {
  Engine& e;
  CallSlot* slot = nullptr;
  explicit SlotLease(Engine& eng) : e(eng) {
    static const int max_in_flight = getenv("QWGPU_MAX_IN_FLIGHT") ? std::max(1, atoi(getenv("QWGPU_MAX_IN_FLIGHT"))) : 16;
    {
      std::unique_lock<std::mutex> g(e.mu);
      e.cv_admit.wait(g, [&] { return e.admitted < max_in_flight; });
      e.admitted++;
      if (!e.free_slots.empty()) { slot = e.free_slots.back(); e.free_slots.pop_back(); }
    }
    if (!slot) {
      try {
        slot = new CallSlot();
        CUDA_CHECK(cudaStreamCreateWithFlags(&slot->stream, cudaStreamNonBlocking));
        for (cudaEvent_t* ev : {&slot->ev0, &slot->ev1, &slot->ev2, &slot->ev3}) CUDA_CHECK(cudaEventCreate(ev));
        CUDA_CHECK(cudaEventCreateWithFlags(&slot->ev_block, cudaEventBlockingSync | cudaEventDisableTiming));
      } catch (...) {
        delete slot;
        { std::lock_guard<std::mutex> g(e.mu); e.admitted--; }
        e.cv_admit.notify_one();
        throw;
      }
    }
    e.in_flight.fetch_add(1);
  }
  // the slot goes back to the pool only once its stream is idle: on an error path copies / kernels of this
  // call may still be in flight, and the next call would reuse the pinned buffers under them
  ~SlotLease() {
    cudaStreamSynchronize(slot->stream);
    e.in_flight.fetch_sub(1);
    {
      std::lock_guard<std::mutex> g(e.mu);
      e.free_slots.push_back(slot);
      e.admitted--;
    }
    e.cv_admit.notify_one();
  }
};

// Waiting for the call's stream: cudaStreamSynchronize spins on a CPU core, which is the fastest wake-up while a
// few calls are in flight (single-query latency) and a disaster when more host threads wait than there are cores
// to spare — the spinners starve the threads that still have plans to compile. Beyond a quarter of the cores the
// wait goes through a blocking event instead (the thread sleeps until the driver's interrupt).
static void wait_call(Engine& e, CallSlot& slot) {
  static const uint32_t spin_limit = getenv("QWGPU_SPIN_LIMIT") ? (uint32_t)atoi(getenv("QWGPU_SPIN_LIMIT")) : std::max(2u, std::thread::hardware_concurrency() / 4);
  if (e.in_flight.load(std::memory_order_relaxed) > (int)spin_limit) {
    CUDA_CHECK(cudaEventRecord(slot.ev_block, slot.stream));
    CUDA_CHECK(cudaEventSynchronize(slot.ev_block));
  } else CUDA_CHECK(cudaStreamSynchronize(slot.stream));
}

// collect / histogram pass flags; F_SAMPLE: a BM25-union collect pass that samples its own threshold
// (k_union<MODE_SAMPLE_COLLECT>, launched cooperatively)
enum { F_REC = 1, F_REFINE = 2, F_CANDS_ONLY = 4, F_SAMPLE = 8 };

// bytes of a split's hit list in its output region (a merged batch keeps the lists in scratch)
static size_t out_hit_bytes(const DSplitPlan& P, bool do_merge) {
  return do_merge ? 0 : (size_t)P.max_hits * (P.score_hits ? sizeof(QwScoreHit) : sizeof(QwHit));
}

// One device run of a lowered batch on the call's slot. lay_out() places every region in the slot's buffers: blob
// (copied to the device: plans, programs, work lists), scratch (device only) and out (copied back); stage() gives the
// run's copies of the plans their addresses and copies the blob over; run() issues the passes.
struct Run {
  Engine& e;
  CallSlot& slot;
  BatchStats& stats;
  const std::vector<Lowered>& low;
  const std::vector<uint32_t>& idx;
  const Route& r;
  const MergeSpec* merge;
  const GatherSpec* gather;
  const bool do_merge, do_gather;
  const uint32_t n;
  const cudaStream_t st;
  std::vector<DSplitPlan> plans;      // copies of the lowered plans with the run's positions, capacities and addresses
  std::vector<uint32_t> bounds_base;  // per split: position of its histogram bounds in the batch's table
  struct Split { size_t out, cand, tr_best, tr_match, h_table, h_keys, h_cells; };  // offsets of a split's regions
  std::vector<Split> at;
  bool any_topk, any_deep, any_trace, any_hashed, any_composite, any_fast_aggs;
  uint32_t kmax, deep_cap, tie_max_n;
  PrePass& pre = slot.pre;  // the batch's pre-pass records
  size_t ts_bm_bytes;  // the bitmap region (term-set nodes)
  size_t o_plans, o_instr, o_cols, o_aggs, o_fwa, o_fws, o_sstr, o_bounds, o_rank, o_smp, o_phr, o_phl, o_pext, o_tsn, o_tst, o_fwd, o_fwds, blob_bytes;
  size_t s_thr, s_hist, s_state, s_wmax, s_sync, s_cand, s_surv, s_deep_m, s_hits, s_cut, s_grecv, s_vblk, s_tsbm, s_trace_state, s_trace_data, s_hash, scratch_bytes;
  size_t rec_bytes, o_merged, o_ghdr, o_final, o_err, out_bytes;
  // the collect pass samples its own threshold (qw_fused_sample_plan): its cooperative grid and per-split sample weights
  bool self_sample;
  uint32_t sample_grid;
  std::vector<uint32_t> sample_stride;
  std::vector<std::vector<DHKey>> h_keys;  // per hashed split: the used cells, copied back
  std::vector<std::vector<QwAggCell>> h_cells;
  KParams kp;
  int occ;
  float main_ms;  // device time of the run's collect passes

  // the work items of k_phrase (pre.phr) or k_phrase_long (pre.phl): the driver blocks of their phrases
  uint32_t phrase_work(const std::vector<DPhrase>& v) const {
    if (v.empty()) return 0;
    const DPhrase& p = v.back();
    return p.first_work + (p.n_terms > QW_MAX_PHRASE_TERMS ? pre.pext[p.exp] : p.t[p.driver]).nblk;
  }
  // the work items of k_term_set: the posting blocks of its terms
  uint32_t term_set_work() const { return pre.tst.empty() ? 0 : pre.tst.back().first_block + pre.tst.back().nblk; }

  // at_bound: every hashed table is sized at its bound (the re-run after an overflow), else at
  // min(bound, QWGPU_HASHED_INIT_CELLS) cells
  void lay_out(bool at_bound) {
    plans.resize(n);
    bounds_base.resize(n);
    at.assign(n, Split{});
    any_topk = any_deep = any_trace = any_hashed = any_composite = any_fast_aggs = false;
    kmax = 1;
    deep_cap = tie_max_n = 0;
    pre.phr.clear(); pre.phl.clear(); pre.pext.clear(); pre.tsn.clear(); pre.tst.clear(); pre.operands.clear();
    ts_bm_bytes = 0;
    size_t vblk_bytes = 0;
    h_keys.assign(n, {});
    h_cells.assign(n, {});
    uint32_t tot_instr = 0, tot_cols = 0, tot_aggs = 0, tot_bounds = 0;
    for (uint32_t i = 0; i < n; i++) {
      const Lowered& L = low[i];
      DSplitPlan& P = plans[i] = L.P;
      P.num_windows = r.fw_all[i + 1] - r.fw_all[i];
      if (do_merge) P.score_hits = 0;  // (k_merge reads QwHit lists)
      P.instr_base = tot_instr; P.col_base = tot_cols; P.agg_base = tot_aggs;
      bounds_base[i] = tot_bounds;
      tot_instr += P.n_instr; tot_cols += P.n_cols; tot_aggs += P.n_aggs; tot_bounds += (uint32_t)L.bounds.size();
      // privatised counters + stats triples must fit the (dead at collect time) staging area
      if (P.fast_aggs && (((size_t)P.n_cells * 4 + 7) & ~(size_t)7) + (size_t)P.n_stat_cells * 24 > stage_bytes_for(r.W)) P.fast_aggs = 0;
      if (P.hashed) {
        any_hashed = true;
        for (const DAgg& d : L.aggs) if (d.comp & QW_AGG_COMP_LEVEL) any_composite = true;
        P.h_cap = (uint32_t)(at_bound ? L.h_bound : std::min<uint64_t>(L.h_bound, QWGPU_HASHED_INIT_CELLS));
        P.h_mask = agg_hashed_slots(P.h_cap) - 1;
      }
      // the plan's pre-pass records in the batch's numbering
      const uint64_t pext0 = pre.pext.size();
      const uint32_t node0 = (uint32_t)pre.tsn.size();
      pre.pext.insert(pre.pext.end(), L.phrase_ext.begin(), L.phrase_ext.end());
      for (DTermSetTerm t : L.ts_terms) {
        t.first_block = term_set_work();
        t.node += node0;
        pre.tst.push_back(t);
      }
      for (const Lowered::Operand& f : L.operands) {
        const uint32_t instr = P.instr_base + f.instr;
        if (f.entry) {
          pre.operands.push_back({instr, PrePass::Operand::ADDR, (uint64_t)f.entry->d_bits});
        } else if (L.instrs[f.instr].op == OP_TERM_SET) {
          // a term set: one doc bitmap
          pre.operands.push_back({instr, PrePass::Operand::BITMAP, ts_bm_bytes});
          pre.tsn.push_back(DTermSetNode{ts_bm_bytes});
          ts_bm_bytes += (size_t)((P.num_docs + 31) / 32) * 4;
        } else {
          // a phrase: one uncompressed posting block per block of its driver term (phrase_kernel.cuh)
          std::vector<DPhrase>& v = L.phrases[f.rec].n_terms > QW_MAX_PHRASE_TERMS ? pre.phl : pre.phr;
          const uint32_t first_work = phrase_work(v);
          v.push_back(L.phrases[f.rec]);
          DPhrase& ph = v.back();
          ph.first_work = first_work;
          ph.out = vblk_bytes;
          ph.exp += pext0;
          vblk_bytes += (size_t)L.instrs[f.instr].n * sizeof(VBlk);
          pre.operands.push_back({instr, PrePass::Operand::VBLK, ph.out});
        }
      }
      kmax = std::max(kmax, P.max_hits);
      any_topk |= P.max_hits > 0;
      if (P.max_hits > QW_MAX_TOPK) { any_deep = true; deep_cap = std::max(deep_cap, qw_cand_cap(P.max_hits)); }
      any_trace |= P.tr_on != 0;
    }
    // BM25-union top-K calls sample the threshold inside the collect pass when the batch qualifies. Cross-rank calls
    // keep the two-launch path: their cooperative grid could queue behind another lane's NCCL kernel that is itself
    // waiting on a peer rank.
    self_sample = false;
    sample_grid = 0;
    if (r.kind == Route::UNION && any_topk && !any_deep && !do_gather && e.coop_launch && r.ulay_s.cap >= QW_HIST_BINS * 4 + 64) {
      int uocc = 0;
      CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&uocc, qwk::k_union<qwk::MODE_SAMPLE_COLLECT>, QU_THREADS, r.ulay_s.total));
      std::vector<uint32_t> mh(n);
      for (uint32_t i = 0; i < n; i++) mh[i] = plans[i].max_hits;
      sample_grid = (uint32_t)(e.sm_count * std::max(uocc, 0));
      sample_stride.assign(n, 1);
      self_sample = qw_fused_sample_plan(r.fw_all.data(), mh.data(), n, sample_grid, sample_stride.data());
    }
    Arena blob{256};
    o_plans = blob.take(n * sizeof(DSplitPlan));
    o_instr = blob.take(tot_instr * sizeof(DInstr));
    o_cols = blob.take(std::max(tot_cols, 1u) * sizeof(DCol));
    o_aggs = blob.take(std::max(tot_aggs, 1u) * sizeof(DAgg));
    o_fwa = blob.take((n + 1) * 4);
    o_fws = blob.take((n + 1) * 4);
    o_sstr = blob.take(self_sample ? (size_t)n * 4 : 0);
    o_bounds = blob.take((size_t)tot_bounds * 8);
    o_rank = blob.take((size_t)n * 4);
    o_smp = blob.take(r.sample_win.size() * 4);
    o_phr = blob.take(pre.phr.size() * sizeof(DPhrase));
    o_phl = blob.take(pre.phl.size() * sizeof(DPhrase));
    o_pext = blob.take(pre.pext.size() * sizeof(DPhraseTerm));
    o_tsn = blob.take(pre.tsn.size() * sizeof(DTermSetNode));
    o_tst = blob.take(pre.tst.size() * sizeof(DTermSetTerm));
    o_fwd = blob.take(r.fw_drv.size() * 4);
    o_fwds = blob.take(r.fw_dsm.size() * 4);
    blob_bytes = blob.off;
    rec_bytes = do_merge ? sizeof(RankHeader) + (size_t)merge->k * sizeof(MergedHit) : 0;  // a merged list
    Arena s{256};
    s_thr = s.take(n * sizeof(DThresh));
    s_hist = s.take((size_t)n * QW_HIST_BINS * 4);
    s_state = s.take((size_t)n * 4);
    s_wmax = s.take(r.rec_l0 ? (size_t)r.fw_all[n] * 2 : 0);
    s_sync = s.take(self_sample ? 4 : 0);  // the grid barrier's counter (zeroed with the prefix below s_cand)
    // candidate lists: qw_cand_cap(K) keys of 24 bytes per split; with a deep plan in the batch, the survivor arrays
    // of the deep selection path mirror them (same offsets from s_surv; used by the deep splits only)
    size_t cand_bytes = 0;
    for (uint32_t i = 0; i < n; i++) { at[i].cand = cand_bytes; cand_bytes += any_topk ? (size_t)qw_cand_cap(plans[i].max_hits) * 24 : 0; }
    s_cand = s.take(cand_bytes);
    s_surv = s.take(any_deep ? cand_bytes : 0);
    s_deep_m = s.take(any_deep ? (size_t)n * 4 : 0);
    s_hits = s.take(do_merge ? (size_t)n * kmax * sizeof(QwHit) : 0);
    s_cut = s.take((size_t)std::max<uint32_t>(n, 64) * 4 + 1024);  // split merge's cut, then the gathered merge's
    s_grecv = s.take(gather && gather->world > 1 && do_merge ? (size_t)gather->world * rec_bytes : 0);
    s_vblk = s.take(vblk_bytes);
    // term-set bitmaps: beyond s_cand, since the exact top-K path clears the prefix again after the pre-pass
    s_tsbm = s.take(ts_bm_bytes);
    // find_trace_ids: per split a DTraceState (one region, set to 0xFF bytes), then best[] + match bitmap (zeroed)
    s_trace_state = s.take(any_trace ? (size_t)n * sizeof(qwk::DTraceState) : 0);
    s_trace_data = s.off;
    for (uint32_t i = 0; i < n; i++)
      if (plans[i].tr_on) {
        at[i].tr_best = s.take((size_t)plans[i].tr_num_ords * 8);
        at[i].tr_match = s.take((size_t)((plans[i].num_docs + 31) / 32) * 4);
      }
    // hashed aggregation cells: per split [slot table][key records][cells]
    s_hash = s.off;
    for (uint32_t i = 0; i < n; i++) {
      const DSplitPlan& P = plans[i];
      if (!P.hashed) continue;
      at[i].h_table = s.take((size_t)(P.h_mask + 1) * 4);
      at[i].h_keys = s.take((size_t)P.h_cap * sizeof(DHKey));
      at[i].h_cells = s.take((size_t)P.h_cap * sizeof(QwAggCell));
    }
    scratch_bytes = s.off;
    Arena o{256};
    for (uint32_t i = 0; i < n; i++)
      at[i].out = o.take(sizeof(DSplitOut) + out_hit_bytes(plans[i], do_merge) + (size_t)plans[i].n_cells * sizeof(QwAggCell));
    o_merged = o.take(rec_bytes);  // the batch's merged top-k = this rank's gather record
    if (do_gather) {
      o_ghdr = o.take((size_t)gather->world * sizeof(RankHeader));  // (compacted copy of the gathered headers)
      o_final = o.take(rec_bytes);
    }
    o_err = o.take(self_sample ? 4 : 0);  // 1: the grid barrier timed out
    out_bytes = o.off;
  }

  // slots are sized to the largest request the context has seen: a slot that meets a bigger request later would
  // have to cudaFree / cudaMalloc (device-synchronising) in the middle of concurrent searches
  void size_slot() {
    size_t want_blob, want_scratch, want_out;
    {
      std::lock_guard<std::mutex> g(e.mu);
      e.hw_blob = std::max(e.hw_blob, blob_bytes); e.hw_scratch = std::max(e.hw_scratch, scratch_bytes); e.hw_out = std::max(e.hw_out, out_bytes);
      // (only while the marks stay moderate: one huge aggregation request must not size every slot after itself)
      auto sized = [](size_t hw, size_t need) { return hw <= ((size_t)64 << 20) ? hw : need; };
      want_blob = sized(e.hw_blob, blob_bytes); want_scratch = sized(e.hw_scratch, scratch_bytes); want_out = sized(e.hw_out, out_bytes);
    }
    slot.ensure(want_blob, want_scratch, want_out);
  }

  // Cross-rank phase (after this rank's result is final: a verification fallback must not repeat a collective the
  // other ranks run once): the rank's record at out + o_merged -> every rank (one NCCL all-gather on the call's
  // stream) -> merged again on the device -> [gathered headers][final hits] copied back
  void exchange() {
    const MergeSpec& m = *merge;
    const GatherSpec& g = *gather;
    uint8_t* g_recv = slot.d_scratch + s_grecv;
    if (g.allgather(g.comm, slot.d_out + o_merged, g_recv, rec_bytes, (void*)st)) fail(QWGPU_EINTERNAL, "ncclAllGather failed");
    const qwk::SrcGathered gsrc{g_recv, (uint32_t)rec_bytes, (uint32_t)sizeof(RankHeader)};
    uint32_t* g_cut = (uint32_t*)(slot.d_scratch + s_cut) + std::max<uint32_t>(n, 64);
    qwk::k_merge_prep<qwk::SrcGathered><<<1, 1024, 0, st>>>(gsrc, (uint32_t)g.world, m.k, m.order1, m.order2, g_cut);
    RankHeader* fin = (RankHeader*)(slot.d_out + o_final);
    qwk::k_merge<qwk::SrcGathered><<<(uint32_t)(((uint64_t)g.world * m.k * 32 + 255) / 256), 256, 0, st>>>(gsrc, g_cut, (uint32_t)g.world, m.k, m.k, m.order1, m.order2,
                                                                                    (MergedHit*)(fin + 1), &fin->n_hits);
    CUDA_CHECK(cudaMemcpy2DAsync(slot.d_out + o_ghdr, sizeof(RankHeader), g_recv, rec_bytes, sizeof(RankHeader), (size_t)g.world, cudaMemcpyDeviceToDevice, st));
    CUDA_CHECK(cudaMemcpyAsync(slot.h_out + o_ghdr, slot.d_out + o_ghdr, out_bytes - o_ghdr, cudaMemcpyDeviceToHost, st));
  }

  // the run's plans get the slot's addresses; everything the kernels read goes to the device in one copy
  void stage() {
    uint8_t *hb = slot.h_blob, *db = slot.d_blob;
    for (uint32_t i = 0; i < n; i++) {
      const Lowered& L = low[i];
      DSplitPlan& P = plans[i];
      any_fast_aggs |= P.fast_aggs != 0;
      if (P.tr_on) tie_max_n = std::max(tie_max_n, P.tr_n);
      DSplitOut* ob = (DSplitOut*)(slot.d_out + at[i].out);
      P.out_num_hits = (uint64_t)&ob->num_hits;  // (the eligible count follows)
      P.out_nhits = (uint64_t)&ob->n_hits;
      P.out_cand_count = (uint64_t)&ob->cand_count;
      P.out_hits = do_merge ? (uint64_t)(slot.d_scratch + s_hits + (size_t)i * kmax * sizeof(QwHit)) : (uint64_t)(ob + 1);
      P.out_cells = (uint64_t)((uint8_t*)(ob + 1) + out_hit_bytes(P, do_merge));
      P.out_hist = (uint64_t)(slot.d_scratch + s_hist + (size_t)i * QW_HIST_BINS * 4);
      P.out_cands = (uint64_t)(slot.d_scratch + s_cand + at[i].cand);
      if (P.tr_on) {
        P.tr_state = (uint64_t)(slot.d_scratch + s_trace_state + (size_t)i * sizeof(qwk::DTraceState));
        P.tr_best = (uint64_t)(slot.d_scratch + at[i].tr_best);
        P.match_out = (uint64_t)(slot.d_scratch + at[i].tr_match);
        P.tr_tie = (uint64_t)&ob->trace_replayed;
      }
      if (P.hashed) {
        P.h_table = (uint64_t)(slot.d_scratch + at[i].h_table);
        P.h_keys = (uint64_t)(slot.d_scratch + at[i].h_keys);
        P.h_cells = (uint64_t)(slot.d_scratch + at[i].h_cells);
        P.h_ctr = (uint64_t)&ob->hashed_cells;
      }
      if (L.fill) P.match_out = (uint64_t)L.fill->d_bits;
      memcpy(hb + o_instr + P.instr_base * sizeof(DInstr), L.instrs.data(), P.n_instr * sizeof(DInstr));
      // (lowering left each column set's table as an index into the split's tables, like the histograms' below)
      DInstr* instrs = (DInstr*)(hb + o_instr) + P.instr_base;
      for (uint32_t k = 0; k < P.n_instr; k++)
        if (instrs[k].op == OP_COL_SET) instrs[k].a = (uint64_t)(db + o_bounds) + (bounds_base[i] + instrs[k].a) * 8;
      memcpy(hb + o_plans + i * sizeof(DSplitPlan), &P, sizeof P);
      if (P.n_cols) memcpy(hb + o_cols + P.col_base * sizeof(DCol), L.cols.data(), P.n_cols * sizeof(DCol));
      DAgg* aggs = (DAgg*)(hb + o_aggs) + P.agg_base;
      if (P.n_aggs) memcpy(aggs, L.aggs.data(), P.n_aggs * sizeof(DAgg));
      // (lowering left each fast-path histogram's and each percentiles node's table as an index into the split's tables)
      for (uint32_t a = 0; a < P.n_aggs; a++)
        if ((P.fast_aggs && aggs[a].kind == QW_AGG_HISTOGRAM) || aggs[a].kind == QW_AGG_PERCENTILES)
          aggs[a].bounds = (uint64_t)(db + o_bounds) + (bounds_base[i] + aggs[a].bounds) * 8;
      if (!L.bounds.empty()) memcpy(hb + o_bounds + (size_t)bounds_base[i] * 8, L.bounds.data(), L.bounds.size() * 8);
    }
    // the pre-pass records and the operands that read their output, offsets turned into addresses
    const uint64_t vblk = (uint64_t)(slot.d_scratch + s_vblk), bm = (uint64_t)(slot.d_scratch + s_tsbm);
    for (auto [o, v] : {std::make_pair(o_phr, &pre.phr), std::make_pair(o_phl, &pre.phl)}) {
      DPhrase* d = (DPhrase*)(hb + o);
      for (size_t k = 0; k < v->size(); k++) {
        d[k] = (*v)[k];
        d[k].out += vblk;
        d[k].exp = (uint64_t)(db + o_pext) + d[k].exp * sizeof(DPhraseTerm);
      }
    }
    if (!pre.pext.empty()) memcpy(hb + o_pext, pre.pext.data(), pre.pext.size() * sizeof(DPhraseTerm));
    for (size_t k = 0; k < pre.tsn.size(); k++) ((DTermSetNode*)(hb + o_tsn))[k].bitmap = bm + pre.tsn[k].bitmap;
    if (!pre.tst.empty()) memcpy(hb + o_tst, pre.tst.data(), pre.tst.size() * sizeof(DTermSetTerm));
    for (const PrePass::Operand& f : pre.operands)
      ((DInstr*)(hb + o_instr))[f.instr].a = f.kind == PrePass::Operand::ADDR ? f.off : (f.kind == PrePass::Operand::VBLK ? vblk : bm) + f.off;
    if (do_merge) for (uint32_t i = 0; i < n; i++) ((uint32_t*)(hb + o_rank))[i] = merge->rank[idx[i]];
    if (!r.sample_win.empty()) memcpy(hb + o_smp, r.sample_win.data(), r.sample_win.size() * 4);
    if (!r.fw_drv.empty()) { memcpy(hb + o_fwd, r.fw_drv.data(), (n + 1) * 4); memcpy(hb + o_fwds, r.fw_dsm.data(), (n + 1) * 4); }
    memcpy(hb + o_fwa, r.fw_all.data(), (n + 1) * 4);
    memcpy(hb + o_fws, r.fw_smp.data(), (n + 1) * 4);
    if (self_sample) memcpy(hb + o_sstr, sample_stride.data(), (size_t)n * 4);
    CUDA_CHECK(cudaMemcpyAsync(db, hb, blob_bytes, cudaMemcpyHostToDevice, st));
    stats.h2d_bytes += blob_bytes;

    kp = KParams{};
    kp.plans = (const DSplitPlan*)(db + o_plans);
    kp.instrs = (const DInstr*)(db + o_instr);
    kp.cols = (const DCol*)(db + o_cols);
    kp.aggs = (const DAgg*)(db + o_aggs);
    kp.thresh = (DThresh*)(slot.d_scratch + s_thr);
    kp.W = r.W;
    kp.stage_bytes = stage_bytes_for(r.W);
    // privatised aggregation counters (and the radix histogram, 8 KB) live in the staging area
    uint32_t max_cells = 0;
    bool any_aggs = false;
    for (const DSplitPlan& P : plans) { max_cells = std::max(max_cells, P.n_cells); any_aggs |= P.n_aggs > 0; }
    kp.smem_aggs = (any_aggs && max_cells * 4 <= kp.stage_bytes && max_cells <= QW_SMEM_AGG_CELLS) ? 1 : 0;
    kp.sm = r.lay;
    kp.wmax = (uint16_t*)(slot.d_scratch + s_wmax);
    kp.split_state = (const uint32_t*)(slot.d_scratch + s_state);
    CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, qwk::k_window<qwk::MODE_COLLECT>, QW_THREADS, r.lay.total));
    occ = std::max(occ, 1);
  }

  // one pass over the batch on the route's kernel when it serves the pass, else on k_window
  void launch(int mode, bool sampled, uint32_t level, uint32_t use_prefix, uint32_t flags) {
    const Route::Kind kind = (flags & F_SAMPLE) || r.serves(mode, level, use_prefix, flags) ? r.kind : Route::WINDOW;
    auto launched = [&](uint32_t kernel) { stats.launches++; stats.kernel_mask |= kernel; };
    // the pass's work list: k_driver walks posting blocks, every other kernel windows
    const bool drv = kind == Route::DRIVER;
    DWorkList wl;
    wl.first_work = (const uint32_t*)(slot.d_blob + (drv ? (sampled ? o_fwds : o_fwd) : (sampled ? o_fws : o_fwa)));
    wl.n_splits = n;
    wl.total_work = drv ? (sampled ? r.fw_dsm[n] : r.fw_drv[n]) : (sampled ? r.fw_smp[n] : r.fw_all[n]);
    wl.stride = sampled ? r.stride : 1;
    if (wl.total_work == 0) return;
    if (drv) {
      qwk::DrvParams d{};
      d.plans = kp.plans; d.instrs = kp.instrs; d.cols = kp.cols; d.thresh = kp.thresh;
      d.wl = wl; d.level = level; d.use_prefix = use_prefix;
      const uint32_t dgrid = std::min<uint32_t>((wl.total_work + QD_WARPS - 1) / QD_WARPS, (uint32_t)(e.sm_count * 4));
      if (mode == qwk::MODE_HIST) qwk::k_driver<qwk::MODE_HIST><<<dgrid, QD_WARPS * 32, 0, st>>>(d);
      else qwk::k_driver<qwk::MODE_COLLECT><<<dgrid, QD_WARPS * 32, 0, st>>>(d);
      launched(QWGPU_KERNEL_DRIVER);
      return;
    }
    if (kind == Route::AGGSCAN) {
      qwk::AParams a{};
      a.plans = kp.plans; a.cols = kp.cols; a.aggs = kp.aggs;
      a.wl = wl;
      a.sm = r.alay;
      int aocc = 1;
      CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&aocc, qwk::k_aggscan, QA_THREADS, r.alay.total));
      const uint32_t agrid = std::min<uint32_t>(wl.total_work, (uint32_t)(e.sm_count * std::max(aocc, 1)));
      qwk::k_aggscan<<<agrid, QA_THREADS, r.alay.total, st>>>(a);
      launched(QWGPU_KERNEL_AGGSCAN);
      return;
    }
    if (kind == Route::UNION) {
      qwk::UParams u{};
      u.plans = kp.plans; u.instrs = kp.instrs; u.cols = kp.cols; u.thresh = kp.thresh;
      u.wl = wl; u.W = sampled ? r.W_h : r.W;
      u.sm = mode == qwk::MODE_HIST ? r.ulay_h : r.ulay_c;
      // cross-rank calls leave a few block slots free: the persistent grid would otherwise hold every SM's shared
      // memory, a concurrent call's NCCL kernel would take the place of one of its blocks, and that block — with its
      // static share of the windows — would only start when another one has finished (twice the kernel time)
      const uint32_t ugrid = std::min<uint32_t>(wl.total_work, (uint32_t)(e.sm_count * QU_MINB) - (do_gather ? 4u : 0u));
      if (flags & F_SAMPLE) {
        // one block per resident slot (occupancy x SMs, checked by qw_fused_sample_plan against the work): the grid
        // barrier after the sample needs every block resident, which only a cooperative launch guarantees
        u.sm = r.ulay_s;
        u.sample_stride = (const uint32_t*)(slot.d_blob + o_sstr);
        u.sync = (uint32_t*)(slot.d_scratch + s_sync);
        u.err = (uint32_t*)(slot.d_out + o_err);
        void* args[] = {&u};
        CUDA_CHECK(cudaLaunchCooperativeKernel((const void*)qwk::k_union<qwk::MODE_SAMPLE_COLLECT>, dim3(sample_grid), dim3(QU_THREADS), args,
                                               u.sm.total, st));
      } else if (mode == qwk::MODE_HIST) qwk::k_union<qwk::MODE_HIST><<<ugrid, QU_THREADS, u.sm.total, st>>>(u);
      else qwk::k_union<qwk::MODE_COLLECT><<<ugrid, QU_THREADS, u.sm.total, st>>>(u);
      launched(QWGPU_KERNEL_UNION);
      return;
    }
    KParams q = kp;
    q.wl = wl;
    q.sample_win = (sampled && r.edge_sample) ? (const uint32_t*)(slot.d_blob + o_smp) : nullptr;
    q.level = level;
    q.use_prefix = use_prefix;
    q.rec_l0 = (flags & F_REC) ? 1 : 0;
    q.refine = (flags & F_REFINE) ? 1 : 0;
    q.cands_only = (flags & F_CANDS_ONLY) ? 1 : 0;
    const uint32_t grid = std::min<uint32_t>(wl.total_work, (uint32_t)(e.sm_count * occ));
    if (mode == qwk::MODE_HIST) qwk::k_window<qwk::MODE_HIST><<<grid, QW_THREADS, r.lay.total, st>>>(q);
    else if (any_hashed) qwk::k_window<qwk::MODE_COLLECT, true><<<grid, QW_THREADS, r.lay.total, st>>>(q);
    else qwk::k_window<qwk::MODE_COLLECT><<<grid, QW_THREADS, r.lay.total, st>>>(q);
    launched(QWGPU_KERNEL_WINDOW);
    // (k_window aggregates on the fast path where the plan's and the launch's flags both allow it)
    if (mode == qwk::MODE_COLLECT && !(flags & F_CANDS_ONLY) && any_fast_aggs && kp.smem_aggs) stats.kernel_mask |= QWGPU_KERNEL_FAST_AGGS;
    if (mode == qwk::MODE_COLLECT && !(flags & F_CANDS_ONLY) && any_hashed) stats.kernel_mask |= QWGPU_KERNEL_HASHED_AGGS;
  }

  // the collect pass and the kernels that finish the split results (composite cut, trace ids, top-K selection, the
  // batch's merge), then the copy-back, waited for; a candidates-only repair keeps the counts and aggregations out
  void collect(uint32_t flags) {
    const bool full = !(flags & F_CANDS_ONLY);
    if (full) {
      CUDA_CHECK(cudaMemsetAsync(slot.d_out, 0, out_bytes, st));
      if (any_trace) {
        CUDA_CHECK(cudaMemsetAsync(slot.d_scratch + s_trace_state, 0xFF, (size_t)n * sizeof(qwk::DTraceState), st));
        CUDA_CHECK(cudaMemsetAsync(slot.d_scratch + s_trace_data, 0, s_hash - s_trace_data, st));
      }
      for (uint32_t i = 0; i < n; i++)
        if (plans[i].hashed) {
          CUDA_CHECK(cudaMemsetAsync(slot.d_scratch + at[i].h_table, 0xFF, (size_t)(plans[i].h_mask + 1) * 4, st));
          CUDA_CHECK(cudaMemsetAsync(slot.d_scratch + at[i].h_cells, 0, (size_t)plans[i].h_cap * sizeof(QwAggCell), st));
        }
    }
    CUDA_CHECK(cudaEventRecord(slot.ev2, st));
    launch(qwk::MODE_COLLECT, false, 0, 0, flags);
    CUDA_CHECK(cudaEventRecord(slot.ev3, st));
    if (any_composite && full) {
      // each composite's first `size` leaves with their chains and sub-aggregation entries, before the copy-back
      qwk::k_composite_cut<<<n, QC_THREADS, 0, st>>>(kp.plans, kp.aggs);
      stats.launches++;
      stats.kernel_mask |= QWGPU_KERNEL_COMPOSITE_CUT;
    }
    if (any_trace && full) {
      // top N of the per-trace maxima; splits whose N-th and (N+1)-th maxima tie replay the reference's selection
      qwk::k_trace_select<<<n, 1024, 0, st>>>(kp.plans);
      qwk::k_trace_replay<<<n, QT_TILE, trace_replay_smem(tie_max_n), st>>>(kp.plans, kp.cols);
      stats.launches += 2;
      stats.kernel_mask |= QWGPU_KERNEL_TRACE_SELECT;
    }
    const uint32_t sel_smem = 3 * 8 * QW_CAND_CAP;  // [all first words | 3 x QW_SEL_MAX survivors] or 3 x all (degenerate ties)
    if (any_topk) { qwk::k_select<<<dim3(QW_SEL_TILES, n), 1024, sel_smem, st>>>(kp.plans, kp.cols); stats.launches++; }
    if (any_deep) {
      // splits with K > QW_MAX_TOPK (k_select left them): cut, tile sort, rank (deep_select_kernel.cuh)
      uint32_t* d_m = (uint32_t*)(slot.d_scratch + s_deep_m);
      const size_t surv_off = s_surv - s_cand;
      qwk::k_deep_cut<<<n, 1024, 0, st>>>(kp.plans, surv_off, d_m);
      qwk::k_deep_sort<<<dim3((deep_cap + QD_TILE - 1) / QD_TILE, n), 1024, 3 * 8 * QD_TILE, st>>>(kp.plans, surv_off, d_m);
      qwk::k_deep_rank<<<dim3(deep_cap / 256, n), 256, 0, st>>>(kp.plans, kp.cols, surv_off, d_m);
      stats.launches += 3;
      stats.kernel_mask |= QWGPU_KERNEL_DEEP_SELECT;
    }
    if (do_merge) {
      uint32_t* d_cut = (uint32_t*)(slot.d_scratch + s_cut);
      RankHeader* rec = (RankHeader*)(slot.d_out + o_merged);
      const qwk::SrcSplits src{kp.plans, (const uint32_t*)(slot.d_blob + o_rank), do_gather ? 1u : 0u};
      qwk::k_merge_prep<qwk::SrcSplits><<<1, 1024, 0, st>>>(src, n, merge->k, merge->order1, merge->order2, d_cut);
      const uint64_t threads = (uint64_t)n * kmax * 32;  // one warp per hit (warps of pruned hits leave at once)
      qwk::k_merge<qwk::SrcSplits><<<(uint32_t)((threads + 255) / 256), 256, 0, st>>>(src, d_cut, n, kmax, merge->k, merge->order1, merge->order2,
                                                          (MergedHit*)(rec + 1), &rec->n_hits);
      stats.launches += 2;
    }
    const size_t back = do_gather ? o_ghdr : out_bytes;  // (gathering: the final hits follow in the cross-rank phase)
    CUDA_CHECK(cudaMemcpyAsync(slot.h_out, slot.d_out, back, cudaMemcpyDeviceToHost, st));
    stats.d2h_bytes += back;
    CUDA_CHECK(cudaEventRecord(slot.ev1, st));
    wait_call(e, slot);
  }

  // a split's candidate set is good when it holds at least min(K, eligible) and did not overflow
  bool verify(std::vector<uint32_t>& state) const {
    bool all = true;
    for (uint32_t i = 0; i < n; i++) {
      state[i] = 0;
      if (low[i].P.max_hits == 0) continue;
      const DSplitOut& ob = *(const DSplitOut*)(slot.h_out + at[i].out);
      const uint64_t eligible = ob.eligible, cand = ob.cand_count;
      if (cand > qw_cand_cap(low[i].P.max_hits) || cand < std::min<uint64_t>(low[i].P.max_hits, eligible)) { state[i] = 1; all = false; }
    }
    return all;
  }

  // exact radix select over the composite key: one histogram pass per 11-bit digit until the
  // candidate set of every split fits its capacity (qw_cand_cap). After a failed sampled threshold with the
  // level-0 histogram on record (refine), level 0 needs no pass at all, only the failing splits are
  // revisited, and windows whose best digit is below the threshold digit are skipped.
  void exact_select(bool refine, std::vector<uint32_t>& state) {
    const uint32_t* d_state = refine ? kp.split_state : nullptr;
    std::vector<DThresh> th(n);
    auto all_done = [&]() {
      for (uint32_t i = 0; i < n; i++) if (low[i].P.max_hits && (!refine || state[i]) && !th[i].done) return false;
      return true;
    };
    uint32_t max_key_bits = 1, level = 0;
    for (const Lowered& L : low) max_key_bits = std::max(max_key_bits, L.P.key.total_bits);
    bool done = false;
    if (refine) {
      CUDA_CHECK(cudaMemcpyAsync(slot.d_scratch + s_state, state.data(), n * 4, cudaMemcpyHostToDevice, st));
      qwk::k_pick<<<n, 256, 0, st>>>(kp.plans, kp.thresh, 0, 0, 1, d_state);
      stats.launches++;
      CUDA_CHECK(cudaMemcpyAsync(th.data(), slot.d_scratch + s_thr, n * sizeof(DThresh), cudaMemcpyDeviceToHost, st));
      wait_call(e, slot);
      done = all_done();
      level = 1;
    } else {
      CUDA_CHECK(cudaMemsetAsync(slot.d_scratch, 0, s_cand, st));
    }
    for (; !done && level * QW_DIGIT_BITS < max_key_bits; level++) {
      CUDA_CHECK(cudaMemsetAsync(slot.d_scratch + s_hist, 0, (size_t)n * QW_HIST_BINS * 4, st));
      launch(qwk::MODE_HIST, false, level, level > 0 ? 1 : 0, refine ? F_REFINE : 0);
      qwk::k_pick<<<n, 256, 0, st>>>(kp.plans, kp.thresh, level, 0, 1, d_state);
      stats.launches++;
      stats.radix_passes++;
      CUDA_CHECK(cudaMemcpyAsync(th.data(), slot.d_scratch + s_thr, n * sizeof(DThresh), cudaMemcpyDeviceToHost, st));
      wait_call(e, slot);
      done = all_done();
    }
    stats.refined = refine ? 1 : 0;
    collect(refine ? (F_REFINE | F_CANDS_ONLY) : 0);
    if (!verify(state)) fail(QWGPU_EINTERNAL, "top-K candidate selection failed verification");
  }

  // device time up to ev1 since ev0, and of the collect pass between ev2 and ev3
  void add_device_time() {
    float ms = 0, main = 0;
    cudaEventElapsedTime(&ms, slot.ev0, slot.ev1);
    cudaEventElapsedTime(&main, slot.ev2, slot.ev3);
    stats.gpu_time_us += ms * 1000.f;
    main_ms += main;
  }

  // The device part of a call: the threshold and collect passes, the hashed copy-back and the cross-rank exchange.
  // False, with nothing returned, when a split's hashed aggregation cells overflowed their capacity.
  bool run(bool at_bound) {
    main_ms = 0;
    CUDA_CHECK(cudaEventRecord(slot.ev0, st));
    CUDA_CHECK(cudaMemsetAsync(slot.d_scratch, 0, s_cand, st));  // thresholds, histograms, refinement state
    if (const uint32_t blocks = phrase_work(pre.phr)) {
      // phrase pre-pass (inside the timed device region): every phrase of the batch becomes a posting list in
      // scratch (beyond s_cand: never cleared), read by every later pass
      uint32_t max_terms = 1;  // (over k_phrase's phrases only: a long phrase does not widen its shared memory)
      bool any_prefix = false;
      for (const DPhrase& ph : pre.phr) { max_terms = std::max(max_terms, ph.n_terms); any_prefix |= ph.n_exp != 0; }
      const size_t psm = (size_t)QP_WARPS * QP_SMEM_WORDS(max_terms) * 4;
      const uint32_t pgrid = (blocks + QP_WARPS - 1) / QP_WARPS;
      const DPhrase* d_phr = (const DPhrase*)(slot.d_blob + o_phr);
      // the suffix stage of phrase prefixes lives in its own instantiation: plain phrases keep the lean kernel
      if (any_prefix) qwk::k_phrase<true><<<pgrid, QP_WARPS * 32, psm, slot.stream>>>(d_phr, (uint32_t)pre.phr.size(), blocks, max_terms);
      else qwk::k_phrase<false><<<pgrid, QP_WARPS * 32, psm, slot.stream>>>(d_phr, (uint32_t)pre.phr.size(), blocks, max_terms);
      stats.launches++;
      stats.kernel_mask |= QWGPU_KERNEL_PHRASE;
    }
    if (const uint32_t blocks = phrase_work(pre.phl)) {
      // long-phrase pre-pass (phrase_kernel.cuh): the same output, shared memory independent of the phrase length
      qwk::k_phrase_long<<<(blocks + QP_WARPS - 1) / QP_WARPS, QP_WARPS * 32, 0, slot.stream>>>(
          (const DPhrase*)(slot.d_blob + o_phl), (uint32_t)pre.phl.size(), blocks);
      stats.launches++;
      stats.kernel_mask |= QWGPU_KERNEL_PHRASE_LONG;
    }
    if (ts_bm_bytes) {
      // term-set pre-pass (inside the timed device region): every term-set node of the batch becomes a doc bitmap in
      // scratch, read by every later pass (cleared for every node, whether or not its terms hold a block)
      CUDA_CHECK(cudaMemsetAsync(slot.d_scratch + s_tsbm, 0, ts_bm_bytes, st));
    }
    if (const uint32_t blocks = term_set_work()) {
      const uint32_t tgrid = std::min<uint32_t>((blocks + QS_WARPS - 1) / QS_WARPS, (uint32_t)e.sm_count * 8);
      qwk::k_term_set<<<tgrid, QS_WARPS * 32, 0, st>>>((const DTermSetTerm*)(slot.d_blob + o_tst), (uint32_t)pre.tst.size(),
                                                       (const DTermSetNode*)(slot.d_blob + o_tsn), blocks);
      stats.launches++;
      stats.kernel_mask |= QWGPU_KERNEL_TERM_SET;
    }
    stats.window_docs = r.kind == Route::DRIVER ? QW_BLOCK_LEN : r.W;
    std::vector<uint32_t> state(n, 0);  // per split: 1 = its sampled threshold failed
    bool ok = true;
    const bool sampled = self_sample || (any_topk && r.stride > 1);
    if (sampled) {
      if (self_sample) {
        // fast path in one pass: the collect pass takes each block's first window as the threshold sample
        stats.sample_stride = r.fw_all[n] / sample_grid;
        collect(F_SAMPLE);
        if (*(const uint32_t*)(slot.h_out + o_err)) fail(QWGPU_EINTERNAL, "k_union: the grid barrier after the threshold sample timed out");
      } else {
        // fast path: threshold from a 1/stride sample of the windows
        stats.sample_stride = r.stride;
        launch(qwk::MODE_HIST, true, 0, 0, 0);
        qwk::k_pick<<<n, 256, 0, st>>>(kp.plans, kp.thresh, 0, r.edge_sample ? 2 : 1, r.stride, nullptr);
        stats.launches++;
        if (r.rec_l0) CUDA_CHECK(cudaMemsetAsync(slot.d_scratch + s_hist, 0, (size_t)n * QW_HIST_BINS * 4, st));
        collect(r.rec_l0 ? F_REC : 0);
      }
      // verified after the collect pass
      ok = verify(state);
      if (!ok) {
        add_device_time();
        stats.exact_fallbacks++;
        CUDA_CHECK(cudaEventRecord(slot.ev0, st));
      }
    }
    if (!any_topk) collect(0);
    else if (!sampled || !ok) exact_select(!ok && r.rec_l0, state);
    // hashed cells: a split that outgrew its capacity sends the batch round again at the bound (before any
    // cross-rank collective, which must run once); otherwise only the used cells come back
    auto used = [&](uint32_t i) { return ((const DSplitOut*)(slot.h_out + at[i].out))->hashed_cells; };
    bool overflow = false;
    for (uint32_t i = 0; i < n; i++) overflow |= plans[i].hashed && (used(i) >> 31);
    if (overflow && at_bound) fail(QWGPU_EINTERNAL, "hashed aggregation cells overflowed their bound");
    if (!overflow) {
      if (any_hashed) {
        for (uint32_t i = 0; i < n; i++) {
          if (!plans[i].hashed) continue;
          const uint32_t nu = std::min(used(i), plans[i].h_cap);
          h_keys[i].resize(nu);
          h_cells[i].resize(nu);
          if (!nu) continue;
          CUDA_CHECK(cudaMemcpyAsync(h_keys[i].data(), slot.d_scratch + at[i].h_keys, (size_t)nu * sizeof(DHKey), cudaMemcpyDeviceToHost, st));
          CUDA_CHECK(cudaMemcpyAsync(h_cells[i].data(), slot.d_scratch + at[i].h_cells, (size_t)nu * sizeof(QwAggCell), cudaMemcpyDeviceToHost, st));
          stats.d2h_bytes += (size_t)nu * (sizeof(DHKey) + sizeof(QwAggCell));
        }
        wait_call(e, slot);
      }
      if (do_gather) {
        qwk::k_rank_header<<<1, 32, 0, st>>>(kp.plans, n, (RankHeader*)(slot.d_out + o_merged), gather->attempted, gather->successful, gather->n_failed);
        exchange();
        CUDA_CHECK(cudaEventRecord(slot.ev1, st));
        wait_call(e, slot);
        stats.launches += 4;
        stats.d2h_bytes += out_bytes - o_ghdr;
      }
      CUDA_CHECK(cudaGetLastError());
    }
    add_device_time();
    stats.main_kernel_us = main_ms * 1000.f;
    return !overflow;
  }
};

// A plan with QW_NODE_CACHE nodes, lowered against the predicate cache: hits read their entries, misses get new
// entries and, in `fills`, one count-only plan each (the subtree's key nodes as the whole query) whose collect pass
// writes the entry. Nested CACHE nodes of a fill plan are lowered as their children.
static Lowered lower_cached(PredCache* pc, const SplitDev& sp, const uint8_t* plan, size_t plan_len, uint32_t max_hits,
                            std::vector<Lowered>& fills) {
  Lowered C;
  C.pc = pc;
  lower_plan(C, sp, plan, plan_len, max_hits);
  for (const std::shared_ptr<PredEntry>& m : C.misses) {
    QwPlanHeader h;
    memset(&h, 0, sizeof h);
    h.magic = QW_PLAN_MAGIC;
    h.version = 1;
    h.num_nodes = (uint32_t)(m->key.size() / sizeof(QwPlanNode));
    h.count_only = 1;
    h.sort[0] = QwSortSpec{QW_SORT_DOCID, QW_ORDER_DESC, 0xFFFFFFFFu, 0};
    h.sort[1] = QwSortSpec{QW_SORT_NONE, QW_ORDER_DESC, 0xFFFFFFFFu, 0};
    std::string fp((const char*)&h, sizeof h);
    fp += m->key;
    Lowered F;
    F.fill = m;
    lower_plan(F, sp, (const uint8_t*)fp.data(), fp.size(), max_hits);
    fills.push_back(std::move(F));
  }
  return C;
}

// Lowers every plan once per call; a split whose plan cannot be lowered fails alone. idx: position of each lowered
// plan in the caller's arrays. pc: the predicate cache when it is enabled; the fill plans of the batch's misses go to
// `fills`.
static std::vector<Lowered> lower_batch(const std::vector<std::shared_ptr<SplitDev>>& sp, const std::vector<const uint8_t*>& plans,
                                        const std::vector<size_t>& plan_lens, std::vector<SplitOutput>& outs, std::vector<uint32_t>& idx,
                                        uint32_t max_hits, PredCache* pc, std::vector<Lowered>& fills) {
  std::vector<Lowered> low;
  low.reserve(sp.size());
  for (uint32_t i = 0; i < (uint32_t)sp.size(); i++) {
    try {
      if (!sp[i]) fail(QWGPU_ENOTFOUND, "split not registered");
      Lowered L;
      lower_plan(L, *sp[i], plans[i], plan_lens[i], max_hits);
      // Route rule: the cache does not remove the work of k_driver's posting-driven walk, so a plan that k_driver
      // serves with its CACHE nodes lowered as their children keeps that lowering. (k_union and k_aggscan plans never
      // read an entry: a scored or ALL / NONE subtree is always lowered as itself.)
      if (pc && L.has_cache && !driver_eligible(L)) {
        std::vector<Lowered> f;
        try {
          Lowered C = lower_cached(pc, *sp[i], plans[i], plan_lens[i], max_hits, f);
          C.stripped = std::make_shared<Lowered>(std::move(L));
          L = std::move(C);
          for (Lowered& x : f) fills.push_back(std::move(x));
        } catch (const Error&) {
          // (a subtree that does not lower on its own: the plan runs without the cache)
        }
      }
      low.push_back(std::move(L));
      idx.push_back(i);
    } catch (const Error& e) {
      outs[i].status = e.code;
      outs[i].error = e.what();
    }
  }
  // a re-run after an overflow sizes every hashed table of the call at its bound: the call's tables together must
  // fit QWGPU_HASHED_MAX_BYTES, else every hashed split of the call fails here, before any launch
  uint64_t total = 0;
  uint32_t n_hashed = 0;
  for (const Lowered& L : low)
    if (L.P.hashed) { total += agg_hashed_table_bytes(L.h_bound); n_hashed++; }
  if (total <= QWGPU_HASHED_MAX_BYTES) return low;
  std::vector<Lowered> keep;
  std::vector<uint32_t> keep_idx;
  for (size_t k = 0; k < low.size(); k++) {
    if (!low[k].P.hashed) { keep.push_back(std::move(low[k])); keep_idx.push_back(idx[k]); continue; }
    char msg[512];
    snprintf(msg, sizeof msg, "split `%s`: the aggregation may create up to %llu buckets; the hashed tables of the call's %u "
             "hashed splits need %llu bytes at their bounds, more than the GPU limit of %llu bytes per call",
             sp[idx[k]]->id.c_str(), (unsigned long long)low[k].h_bound, n_hashed, (unsigned long long)total,
             (unsigned long long)QWGPU_HASHED_MAX_BYTES);
    outs[idx[k]].status = QWGPU_EUNSUPPORTED;
    outs[idx[k]].error = msg;
  }
  idx.swap(keep_idx);
  return keep;
}

static void strip_doc_key(QwHit& h) { h.flags &= ~1u; h.v1 = 0; }  // (the doc-id sort key's internal fields)

// the QwHit that k_select writes for a hit ranked by _score descending alone
static QwHit expand_score_hit(const QwScoreHit& s) {
  QwHit h;
  h.v1 = f64_to_u64((double)s.score);
  h.v2 = 0;
  h.doc_id = s.doc_id;
  h.flags = 1;
  h.score = s.score;
  h.reserved = 0;
  return h;
}

// one split's result out of its region of the copied-back buffer (and its hashed entries); P: the run's copy of
// the split's plan
static void unpack_split(SplitOutput& o, BatchStats& stats, const Lowered& L, const DSplitPlan& P, const SplitDev& s, const uint8_t* plan,
                         const DSplitOut* ob, bool do_merge, const std::vector<DHKey>& keys, const std::vector<QwAggCell>& cells) {
  o.num_hits = ob->num_hits;
  const uint32_t nh = ob->n_hits;
  const uint8_t* hits = (const uint8_t*)(ob + 1);
  if (!do_merge && P.score_hits) {
    const QwScoreHit* sh = (const QwScoreHit*)hits;
    o.hits.resize(nh);
    for (uint32_t j = 0; j < nh; j++) o.hits[j] = expand_score_hit(sh[j]);
  } else if (!do_merge) {
    o.hits.assign((const QwHit*)hits, (const QwHit*)hits + nh);
    if (P.key.kind[0] == QW_SORT_DOCID) for (auto& h : o.hits) strip_doc_key(h);
  }
  const QwAggCell* c = (const QwAggCell*)(hits + out_hit_bytes(P, do_merge));
  o.cells.assign(c, c + P.n_cells);
  for (auto& cell : o.cells) cell.min_mapped = ~cell.min_mapped;  // device keeps max(~m); see agg_stats
  if (P.hashed) {
    o.hashed = true;
    o.entries.resize(keys.size());
    for (size_t e = 0; e < o.entries.size(); e++) {
      QwAggEntry& x = o.entries[e];
      x.node = keys[e].node_flags & 0xFFu;
      x.flags = keys[e].node_flags >> 8;
      x.parent = keys[e].parent;
      x.key = keys[e].key;
      x.reserved = 0;
      x.cell = cells[e];
      x.cell.min_mapped = ~x.cell.min_mapped;
    }
  }
  if (P.tr_on) {
    if (ob->trace_replayed) stats.kernel_mask |= QWGPU_KERNEL_TRACE_REPLAY;
    // a matched doc without a trace id reads ordinal 0: with an empty dictionary the reference's ord_to_bytes fails
    const QwImgColumn& tc = s.view.columns[L.tr_img_col];
    for (const QwAggCell& cell : o.cells)
      if (cell.count == 1 && cell.sum_bits >= tc.dict_num_terms) {
        o.status = QWGPU_EINTERNAL;
        o.error = "failed to look up a trace id in the column term dictionary";
        o.cells.clear();
        break;
      }
  }
  o.postings_scored = L.postings;
  // SURVEY.md §8d algorithmic bytes: postings (+ fieldnorms, added at lowering) + column probes
  uint64_t bytes = L.alg_bytes;
  auto col_bytes = [&](uint32_t c, uint64_t probes) {
    const QwImgColumn& ic = s.view.columns[c];
    uint64_t full = ((uint64_t)ic.num_vals * ic.bits + 7) / 8;
    return std::min<uint64_t>(probes * ((ic.bits + 7) / 8), full);
  };
  uint64_t driver = L.min_required_df == ~0ull ? P.num_docs : L.min_required_df;
  for (auto& rc : L.range_cols) bytes += col_bytes(rc.first, driver);
  const QwPlanHeader* ph = (const QwPlanHeader*)plan;
  for (int k = 0; k < 2; k++)
    if (ph->sort[k].kind == QW_SORT_COLUMN && ph->sort[k].column != 0xFFFFFFFFu && P.max_hits) bytes += col_bytes(ph->sort[k].column, o.num_hits);
  const QwAggNode* an = (const QwAggNode*)(plan + sizeof(QwPlanHeader) + (size_t)ph->num_nodes * sizeof(QwPlanNode));
  for (uint32_t a = 0; a < ph->num_aggs; a++) if (an[a].column != 0xFFFFFFFFu) bytes += col_bytes(an[a].column, o.num_hits);
  o.algorithmic_bytes = bytes;
}

// The hits of a device-merged list. A batch's own merge names positions in `low`, which `idx` maps back to the
// caller's arrays; a cross-rank merge (idx null) carries GLOBAL split ranks (the caller owns the rank -> split id
// table), and a rank with no searchable split does not know the sort.
static void unpack_merged(const RankHeader* list, const std::vector<Lowered>& low, const std::vector<uint32_t>* idx,
                          std::vector<MergedHit>& merged) {
  const MergedHit* mh = (const MergedHit*)(list + 1);
  merged.assign(mh, mh + list->n_hits);
  for (MergedHit& m : merged) {
    const Lowered* L = idx ? &low[m.split] : low.empty() ? nullptr : &low[0];
    if (idx) m.split = (*idx)[m.split];
    if (L && L->P.key.kind[0] == QW_SORT_DOCID) strip_doc_key(m.hit);
  }
}

// A rank with no searchable split still takes part in the collective, with an empty record (and reports no device work)
static void exchange_empty(Engine& e, const MergeSpec& merge, const GatherSpec& gather, std::vector<MergedHit>& merged,
                           std::vector<RankHeader>& rank_headers) {
  SlotLease lease(e);
  const std::vector<Lowered> none;
  const std::vector<uint32_t> no_idx;
  const Route no_route{};
  BatchStats unused;
  Run run{e, *lease.slot, unused, none, no_idx, no_route, &merge, &gather, true, true, 0, lease.slot->stream};
  run.lay_out(false);
  run.size_slot();
  CUDA_CHECK(cudaMemsetAsync(run.slot.d_out, 0, run.out_bytes, run.st));
  RankHeader h{};
  h.attempted = gather.attempted;
  h.successful = gather.successful;
  h.n_failed = gather.n_failed;
  CUDA_CHECK(cudaMemcpyAsync(run.slot.d_out + run.o_merged, &h, sizeof h, cudaMemcpyHostToDevice, run.st));
  run.exchange();
  wait_call(e, run.slot);
  unpack_merged((const RankHeader*)(run.slot.h_out + run.o_final), none, nullptr, merged);
  const RankHeader* hdrs = (const RankHeader*)(run.slot.h_out + run.o_ghdr);
  rank_headers.assign(hdrs, hdrs + gather.world);
}

void Engine::search(const std::vector<std::shared_ptr<SplitDev>>& sp, const std::vector<const uint8_t*>& plans,
                    const std::vector<size_t>& plan_lens, std::vector<SplitOutput>& outs, BatchStats& stats,
                    const MergeSpec* merge, std::vector<MergedHit>* merged, const GatherSpec* gather, std::vector<RankHeader>* rank_headers) {
  outs.assign(sp.size(), SplitOutput());
  static const bool trace = getenv("QWGPU_TRACE") != nullptr;  // host phase timings on stderr
  using tclock = std::chrono::steady_clock;
  const auto t_begin = tclock::now();
  CUDA_CHECK(cudaSetDevice(device));
  std::vector<uint32_t> idx;
  PredCache* pc = nullptr;
  {
    std::lock_guard<std::mutex> g(pred.mu);
    if (pred.budget) pc = &pred;
  }
  // (declared before the slot lease: the entries they pin are released only once the call's stream is idle)
  std::vector<Lowered> fills;
  std::vector<Lowered> low = lower_batch(sp, plans, plan_lens, outs, idx, max_hits.load(std::memory_order_relaxed), pc, fills);
  const bool gathering = merge && merged && merge->k > 0 && gather && gather->allgather && gather->world > 1 && rank_headers;
  if (low.empty()) {
    if (gathering) exchange_empty(*this, *merge, *gather, *merged, *rank_headers);
    return;
  }
  const auto t_lowered = tclock::now();
  Route r = choose_route(low, max_smem_optin, sm_count);
  // device-side cross-split merge: the per-split hit lists stay in scratch, only the merged top-K comes back
  const bool do_merge = merge && merged && merge->k > 0 && merge->rank.size() == sp.size() &&
                        std::any_of(low.begin(), low.end(), [](const Lowered& L) { return L.P.max_hits > 0; });
  SlotLease lease(*this);
  pred.free_released(lease.slot->stream);
  if (!fills.empty()) {
    // the entries' bitmaps, stream-ordered from the pool. The budget is a ceiling, not a reservation: when the device
    // cannot provide a bitmap, the plans that needed it run without the cache (their stripped lowering) and their
    // other fills are dropped — the optional cache never fails a search
    const cudaStream_t st = lease.slot->stream;
    for (Lowered& F : fills)
      if (cudaMallocFromPoolAsync(&F.fill->d_bits, F.fill->bytes, (cudaMemPool_t)pred.pool, st) != cudaSuccess) {
        cudaGetLastError();
        F.fill->d_bits = nullptr;
      }
    bool fell_back = false;
    for (Lowered& L : low)
      if (std::any_of(L.misses.begin(), L.misses.end(), [](const std::shared_ptr<PredEntry>& m) { return !m->d_bits; })) {
        Lowered s = std::move(*L.stripped);
        L = std::move(s);
        fell_back = true;
      }
    if (fell_back) r = choose_route(low, max_smem_optin, sm_count);
    // (a fill whose entry no plan reads any more is the only holder of it)
    fills.erase(std::remove_if(fills.begin(), fills.end(), [](const Lowered& F) { return !F.fill->d_bits || F.fill.use_count() == 1; }),
                fills.end());
    pred.free_released(st);
  }
  if (!fills.empty()) {
    // the predicate-cache fill pass: every miss of the call as one count-only batch on k_window, before the call's
    // own passes; each entry is zeroed first (windows that a fill plan skips as empty write nothing)
    const cudaStream_t st = lease.slot->stream;
    for (Lowered& F : fills) CUDA_CHECK(cudaMemsetAsync(F.fill->d_bits, 0, F.fill->bytes, st));
    std::vector<uint32_t> fidx(fills.size());
    for (uint32_t i = 0; i < (uint32_t)fills.size(); i++) fidx[i] = i;
    const Route fr = choose_route(fills, max_smem_optin, sm_count, true);
    Run fill{*this, *lease.slot, stats, fills, fidx, fr, nullptr, nullptr, false, false, (uint32_t)fills.size(), st};
    fill.lay_out(false);
    fill.size_slot();
    fill.stage();
    fill.run(false);
    stats.kernel_mask |= QWGPU_KERNEL_PREDICATE_FILL;
  }
  Run run{*this, *lease.slot, stats, low, idx, r, merge, gather, do_merge, do_merge && gathering, (uint32_t)low.size(), lease.slot->stream};
  tclock::time_point t_staged;
  for (bool at_bound : {false, true}) {
    run.lay_out(at_bound);
    run.size_slot();
    run.stage();
    if (!at_bound) t_staged = tclock::now();
    if (run.run(at_bound)) break;
    // a split's hashed aggregation cells outgrew QWGPU_HASHED_INIT_CELLS: the batch runs again with every hashed
    // split's table at its bound, where it cannot overflow (the first run's device time stays in the stats)
    stats.kernel_mask |= QWGPU_KERNEL_HASHED_AGGS_RETRY;
  }

  // the call has finished: its filled entries become visible to other calls
  for (uint32_t i = 0; i < low.size(); i++)
    for (const std::shared_ptr<PredEntry>& m : low[i].misses) pred.publish(sp[idx[i]].get(), m);
  const auto t_searched = tclock::now();
  const uint8_t* h_out = lease.slot->h_out;
  for (uint32_t i = 0; i < low.size(); i++)
    unpack_split(outs[idx[i]], stats, low[i], run.plans[i], *sp[idx[i]], plans[idx[i]], (const DSplitOut*)(h_out + run.at[i].out), do_merge, run.h_keys[i], run.h_cells[i]);
  if (run.do_gather) {
    // the cross-rank result: hits carry GLOBAL split ranks (the caller owns the rank -> split id table)
    unpack_merged((const RankHeader*)(h_out + run.o_final), low, nullptr, *merged);
    const RankHeader* hdrs = (const RankHeader*)(h_out + run.o_ghdr);
    rank_headers->assign(hdrs, hdrs + gather->world);
  } else if (do_merge) {
    unpack_merged((const RankHeader*)(h_out + run.o_merged), low, &idx, *merged);
  }
  if (trace) {
    // (a call re-run after a hashed overflow counts the re-run's staging in launch+wait)
    auto us =[](tclock::time_point a, tclock::time_point b) { return (long)std::chrono::duration_cast<std::chrono::microseconds>(b - a).count(); };
    fprintf(stderr, "[qwgpu] search: lower %ld us, stage %ld us, launch+wait %ld us (device %.0f us), unpack %ld us\n", us(t_begin, t_lowered),
            us(t_lowered, t_staged), us(t_staged, t_searched), stats.gpu_time_us, us(t_searched, tclock::now()));
  }
}

}  // namespace qw
