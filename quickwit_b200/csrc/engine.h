// engine.h — host-side engine: split residency in HBM + batched plan execution on the GPU.
#pragma once
#include <condition_variable>
#include <atomic>
#include <map>
#include <memory>
#include <mutex>
#include <thread>
#include <string>
#include <vector>

#include "common.h"

namespace qw {

struct SplitDev {
  std::string id;
  std::vector<uint8_t> dir;  // host copy of the image up to data_off (headers, dictionary, strings)
  ImageView view;            // over `dir` (view.data is NOT valid on the host)
  uint8_t* d_data = nullptr; // device copy of the data region
  float* d_tabs = nullptr;   // device float[num_fields][256] BM25 norm tables
  uint64_t data_len = 0;
  std::vector<uint8_t> ids16;  // per column: 1 = a bytes column whose dictionary holds only 16-byte values
  // residency: recency for the LRU, state of an asynchronous upload (0 loading, 1 ready, 2 failed)
  uint64_t last_use = 0;
  int state = 1;
  std::string load_error;
  ~SplitDev();
};

struct CallSlot;  // per-call stream + scratch (engine.cu)

struct SplitOutput {
  uint64_t num_hits = 0;
  std::vector<QwHit> hits;
  std::vector<QwAggCell> cells;
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
struct MergedHit {
  QwHit hit;
  uint32_t split;  // index into the caller's split array
  uint32_t pad;
};
// Cross-rank exchange standing in for the root merge (SURVEY.md 8e): after the batch's own device merge the
// rank's fixed-size record {header, best k hits tagged with GLOBAL split ranks} is all-gathered over NCCL on
// the call's stream and the gathered lists are merged on the device again; every rank ends up with the same
// global top-k. `allgather` is ncclAllGather bound to the context's communicator (comm.cpp).
struct RankHeader {  // 64 bytes, written on the device
  uint32_t n_hits, pad;
  uint64_t num_hits, attempted, successful, n_failed, reserved[3];
};
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
  std::condition_variable loaded_cv;
  struct Loader { std::thread t; std::shared_ptr<SplitDev> sp; };
  std::vector<Loader> loaders;
  int sm_count = 0;  // set from cudaDeviceProp in Engine::Engine
  int max_smem_optin = 0;

  explicit Engine(int dev);
  ~Engine();
  void register_split(const char* id, const uint8_t* img, uint64_t len);
  // returns at once; `img` must stay valid until wait_split(id) has returned
  void register_split_async(const char* id, const uint8_t* img, uint64_t len);
  void wait_split(const char* id);  // throws the upload's error, if any
  void set_budget(uint64_t bytes);
  void unregister_split(const char* id);
  std::shared_ptr<SplitDev> find(const std::string& id);
  // Runs plan[i] on splits[i]; fills outs[i] (status per split). Throws only on whole-call errors.
  void search(const std::vector<std::shared_ptr<SplitDev>>& sp, const std::vector<const uint8_t*>& plans,
              const std::vector<size_t>& plan_lens, std::vector<SplitOutput>& outs, BatchStats& stats,
              const MergeSpec* merge = nullptr, std::vector<MergedHit>* merged = nullptr,
              const GatherSpec* gather = nullptr, std::vector<RankHeader>* rank_headers = nullptr);
};

// plan validation helper shared with the compiler: total agg cells + per-node bases
uint64_t agg_cell_layout(const QwAggNode* aggs, uint32_t n, std::vector<uint32_t>* bases);

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
