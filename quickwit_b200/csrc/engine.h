// engine.h — host-side engine: split residency in HBM + batched plan execution on the GPU.
#pragma once
#include <condition_variable>
#include <atomic>
#include <list>
#include <map>
#include <memory>
#include <mutex>
#include <thread>
#include <unordered_map>
#include <string>
#include <vector>

#include "common.h"
#include "device_types.h"

namespace qw {

struct SplitDev;
struct PredCache;

// One predicate-cache entry: the doc set of a QW_NODE_CACHE subtree on one split, as uint32[ceil(num_docs / 32)] in
// HBM. A call holds a reference to every entry it lowered against (a pin: eviction skips entries referenced
// elsewhere); the last reference hands the bitmap back to the cache's pool.
struct PredEntry {
  PredCache* owner = nullptr;
  std::string key;            // the subtree as plan nodes (pred_key)
  void* d_bits = nullptr;     // allocated on the stream of the call that fills it
  uint64_t bytes = 0, last_use = 0;
  ~PredEntry();
};

// The context's predicate cache (DESIGN.md §4.9): the entries of every resident split, LRU within a byte budget.
// Entries are published per split once the call that filled them has finished.
struct PredCache {
  std::mutex mu;  // guards everything below except `used` and the free list; never held while taking Engine::mu
  uint64_t budget = 0, tick = 0;
  uint64_t hits = 0, misses = 0, fills = 0, evictions = 0;
  std::map<const SplitDev*, std::unordered_map<std::string, std::shared_ptr<PredEntry>>> by_split;
  void* pool = nullptr;  // cudaMemPool_t, created with the first non-zero budget
  std::atomic<uint64_t> used{0};  // bytes of every live entry, published or not
  std::mutex free_mu;
  std::vector<void*> to_free;  // bitmaps of released entries, freed stream-ordered by the next call
  // a published entry for `key` (a hit, pinned), else a new unpublished entry of `bytes` (a miss); null when the
  // miss does not fit the budget
  std::shared_ptr<PredEntry> acquire(const SplitDev* sp, const std::string& key, uint64_t bytes, bool* hit);
  void publish(const SplitDev* sp, const std::shared_ptr<PredEntry>& e);  // the first entry published for a key wins
  bool evict_to(uint64_t limit);
  void drop_split(const SplitDev* sp);
  void free_released(void* stream);  // cudaFreeAsync of the released bitmaps on `stream`
};

// The context's partial-result cache (LeafSearchCache, quickwit-search/src/leaf_cache.rs:27-117; DESIGN.md §7.1): the
// encoded LeafSearchResponse of a successful split search, keyed by the split and the normalised per-split request
// (leaf_cache_key, leaf.cpp). LRU within a budget of encoded response bytes, like MemorySizedCache (keys are not
// counted). Host memory only: an entry outlives the split's residency, and registering a split id again or
// unregistering it drops its entries.
struct LeafCache {
  struct Entry {
    std::string key, split_id, value;
  };
  std::mutex mu;  // guards everything below; taken under Engine::mu (never the other way round), and held only for
                  // map updates and copies, never during a search or a merge
  uint64_t budget = 0, used = 0;
  uint64_t hits = 0, misses = 0, fills = 0, evictions = 0;
  std::list<Entry> lru;  // most recently used first
  std::unordered_map<std::string, std::list<Entry>::iterator> index;
  bool on() {
    std::lock_guard<std::mutex> g(mu);
    return budget != 0;
  }
  bool get(const std::string& key, std::string* value);  // true and the entry's bytes on a hit
  // stores unless the value alone exceeds the budget; the caller holds Engine::mu and has checked that the split
  // the value was computed on is still the registered one
  void put(const std::string& split_id, const std::string& key, std::string value);
  void set_budget(uint64_t bytes);
  void drop_split(const std::string& split_id);
};

struct SplitDev {
  std::string id;
  std::vector<uint8_t> dir;  // host copy of the image up to data_off (headers, dictionary, strings)
  ImageView view;            // over `dir` (view.data is NOT valid on the host)
  uint8_t* d_data = nullptr; // device copy of the data region
  float* d_tabs = nullptr;   // device float[num_fields][256] BM25 norm tables
  uint64_t data_len = 0;
  std::vector<uint8_t> ids16;  // per column: 1 = a bytes column whose dictionary holds only 16-byte values
  // per column: the percentiles boundary table (ddsketch.h column_table), built by the first search that needs it
  mutable std::mutex pct_mu;
  mutable std::map<uint32_t, std::shared_ptr<const std::vector<uint64_t>>> pct_tables;
  // residency: recency for the LRU, state of an asynchronous upload (0 loading, 1 ready, 2 failed)
  uint64_t last_use = 0;
  int state = 1;
  std::string load_error;
  PredCache* pred = nullptr;  // the context's predicate cache: this split's entries go with it
  ~SplitDev();
};

struct CallSlot;  // per-call stream + scratch (engine.cu)

struct SplitOutput {
  uint64_t num_hits = 0;
  std::vector<QwHit> hits;
  std::vector<QwAggCell> cells;
  bool hashed = false;              // the plan took the hashed layout: `entries` holds its result, `cells` is empty
  std::vector<QwAggEntry> entries;
  int status = 0;
  std::string error;
  uint64_t postings_scored = 0;
  uint64_t algorithmic_bytes = 0;
};
// Cross-split merge on the device (leaf-level merge of collector.rs:1195-1313 for seam A): when given, the
// per-split top-K lists never leave the GPU; the batch returns its best `k` hits in the leaf's total order
// (sort values in the request's directions, then split id, then doc id in the direction of the first key).
struct MergeSpec {
  uint32_t k = 0;
  uint32_t order1 = QW_ORDER_DESC, order2 = QW_ORDER_DESC;
  std::vector<uint32_t> rank;  // per input split: rank of its split id among the batch's split ids
};
// Cross-rank exchange standing in for the root merge (SURVEY.md 8e): after the batch's own device merge the
// rank's fixed-size record {header, best k hits tagged with GLOBAL split ranks} is all-gathered over NCCL on
// the call's stream and the gathered lists are merged on the device again; every rank ends up with the same
// global top-k. `allgather` is ncclAllGather bound to the context's communicator (comm.cpp).
struct GatherSpec {
  int world = 1, rank = 0;
  // (sendbuf, recvbuf, bytes per rank, stream) -> 0 on success
  int (*allgather)(void* comm, const void* send, void* recv, size_t bytes, void* stream) = nullptr;
  void* comm = nullptr;
  uint64_t attempted = 0, successful = 0, n_failed = 0;  // this rank's split accounting for the header
};
struct BatchStats {
  float gpu_time_us = 0;
  float main_kernel_us = 0;
  uint32_t launches = 0;
  uint32_t exact_fallbacks = 0;
  uint64_t h2d_bytes = 0, d2h_bytes = 0;
  // the path the call took (qwgpu_split_result)
  uint32_t kernel_mask = 0;    // QWGPU_KERNEL_*
  uint32_t window_docs = 0;
  uint32_t sample_stride = 0;  // 0: no sampled threshold pass
  uint32_t radix_passes = 0;   // exact histogram + k_pick rounds
  uint32_t refined = 0;        // 1: candidates-only repair of a failed sampled threshold
};

struct Engine {
  int device = -1;
  std::mutex mu;
  PredCache pred;  // (declared before `splits`: a split's destructor drops its entries here)
  LeafCache leaf;  // off until qwgpu_set_leaf_cache_budget
  std::map<std::string, std::shared_ptr<SplitDev>> splits;
  std::vector<CallSlot*> free_slots;
  std::atomic<int> in_flight{0};  // searches between slot acquisition and release
  int admitted = 0;               // searches past the admission gate (guarded by mu)
  std::condition_variable cv_admit;
  size_t hw_blob = 0, hw_scratch = 0, hw_out = 0;  // largest per-call buffers requested so far (slot sizing)
  uint64_t resident = 0;
  // residency manager: byte budget for the data regions of the resident splits (0 = no limit). Registering a
  // split beyond it evicts the least recently searched splits that no call is using (the counterpart of the
  // searcher's split cache, quickwit-storage split_cache + leaf.rs:210-251 open_split_bundle: a leaf keeps hot
  // splits local and drops cold ones). Uploads can run in the background (register_split_async): `find` waits
  // for a split that is still loading.
  uint64_t budget = 0, tick = 0, evictions = 0;
  // largest max_hits + start_offset a plan may ask for (qwgpu_set_max_hits): QW_MAX_TOPK unless the caller raised it,
  // up to QW_MAX_HITS. Above QW_MAX_TOPK a call needs call-slot scratch that grows with K and stays allocated.
  std::atomic<uint32_t> max_hits{4096};  // (QW_MAX_TOPK)
  std::condition_variable loaded_cv;
  struct Loader { std::thread t; std::shared_ptr<SplitDev> sp; };
  std::vector<Loader> loaders;
  int sm_count = 0;  // set from cudaDeviceProp in Engine::Engine
  int max_smem_optin = 0;
  bool coop_launch = false;  // cudaDevAttrCooperativeLaunch: k_union may sample its own threshold (grid barrier)

  explicit Engine(int dev);
  ~Engine();
  void register_split(const char* id, const uint8_t* img, uint64_t len);
  // returns at once; `img` must stay valid until wait_split(id) has returned
  void register_split_async(const char* id, const uint8_t* img, uint64_t len);
  void wait_split(const char* id);  // throws the upload's error, if any
  void set_budget(uint64_t bytes);
  // predicate cache budget (0 disables the cache and frees every entry that no call is using)
  void set_pred_budget(uint64_t bytes);
  void unregister_split(const char* id);
  std::shared_ptr<SplitDev> find(const std::string& id);
  // Runs plan[i] on splits[i]; fills outs[i] (status per split). Throws only on whole-call errors.
  void search(const std::vector<std::shared_ptr<SplitDev>>& sp, const std::vector<const uint8_t*>& plans,
              const std::vector<size_t>& plan_lens, std::vector<SplitOutput>& outs, BatchStats& stats,
              const MergeSpec* merge = nullptr, std::vector<MergedHit>* merged = nullptr,
              const GatherSpec* gather = nullptr, std::vector<RankHeader>* rank_headers = nullptr);
};

}  // namespace qw

namespace qw { struct Comm; }
struct qwgpu_ctx {
  std::unique_ptr<qw::Engine> engine;  // null for host-only contexts
  // NCCL communicators + the global split table (comm.cpp). One communicator per LANE: the collectives of one
  // communicator must be issued in the same order on every rank, so concurrent searches (one host thread each)
  // take one lane each. comm == lanes[0]; null until qwgpu_comm_init.
  qw::Comm* comm = nullptr;
  qw::Comm* lanes[16] = {nullptr};
  ~qwgpu_ctx();
};
