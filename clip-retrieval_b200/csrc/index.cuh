// The index handle behind b200_index* (flat and IVF-Flat share the row store and the top-k tail).
#pragma once
#include "common.cuh"
#include <map>
#include <mutex>
#include <vector>

struct b200_index {
  int d = 0;
  int device = 0;
  int sms = 132;
  int64_t ntotal = 0;
  int64_t capacity = 0;     // rows allocated in `rows`
  bool reserved = false;
  __half* rows = nullptr;   // flat: insertion order.  IVF: list order after finalize.
  int64_t id_base = 0;
  bool use_staged = true;   // FMA scan through the cp.async.bulk shared-memory ring (knn_scan.cu)
  bool use_mma = true;      // batched queries go through the wgmma scan (knn_mma.cu)
  bool use_hi_only = true;  // > 128 queries: approximate hi-only pass + exact re-score + proof (knn_mma.cu)
  int last_hi_only_fallbacks = 0;   // queries of the last batched search whose proof failed (re-run split)
  const __half* norm_rows[2] = {nullptr, nullptr};   // cache of max_row ||x||^2 per scanned table
  int64_t norm_n[2] = {0, 0};
  float* norm_bound[2] = {nullptr, nullptr};
  int norm_next = 0;

  // IVF-Flat
  int nlist = 0;            // 0 = flat
  int nprobe = 1;
  __half* centroids = nullptr;      // [nlist, d] fp16
  int64_t* list_offsets = nullptr;  // device [nlist + 1] (row offsets into `rows`)
  uint32_t* row_ids = nullptr;      // device [ntotal]: local insertion id of the row at each slot
  std::vector<int64_t> h_list_offsets;
  int64_t nfinal = 0;               // rows already bucketed
  __half* pending = nullptr;        // rows added but not yet bucketed (insertion order)
  int64_t npending = 0, pending_cap = 0;
  int64_t max_list = 0;
  std::vector<uint32_t> pending_lists;   // explicit list of every pending row (0xFFFFFFFF: assign by max inner product)
  uint32_t* id_to_slot = nullptr;         // device [ntotal]: inverse of row_ids, built on the first reconstruct-by-id
  int64_t id_to_slot_n = -1;

  // scratch
  void* ws[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // 0: scan internals; 1..3: callers; 4,5: hi-only mode
  size_t ws_bytes[6] = {0, 0, 0, 0, 0, 0};
  std::mutex mu;             // every search entry (host and device) holds it while it enqueues work
  cudaEvent_t scratch_ev = nullptr;   // recorded after the last search's launches: the next search on ANOTHER
  cudaStream_t scratch_stream = nullptr;   // stream waits on it before it reuses ws[] / norm_bound[]
  bool scratch_used = false;

  // Serving shape (nq <= 4: clip_back.py:362 issues one query): the launches of a search are captured once per
  // (nq, k, nprobe, reconstruct) into a CUDA graph over fixed buffers and replayed; any mutation of the index bumps
  // graph_epoch and the stale graphs are rebuilt.
  struct SearchGraph { cudaGraphExec_t exec = nullptr; int seen = 0; int kernels = 0; uint64_t epoch = 0; };
  std::map<uint64_t, SearchGraph> graphs;
  uint64_t graph_epoch = 1;
  bool use_graphs = true;     // B200_GRAPHS=0 disables
  cudaStream_t cap_stream = nullptr;
  bool capturing = false;     // timing events are recorded as external event nodes while a graph is captured
  float* g_q = nullptr; float* g_D = nullptr; int64_t* g_I = nullptr; float* g_R = nullptr;
  size_t g_q_cap = 0, g_k_cap = 0, g_r_cap = 0;

  // scan timing (CUDA events on the launching stream)
  std::vector<cudaEvent_t> ev;   // pairs
  int ev_used = 0;
  int last_scan_launches = 0;
};

namespace b200 {
inline cudaError_t index_record(b200_index* idx, cudaEvent_t e, cudaStream_t st) {
  return idx->capturing ? cudaEventRecordWithFlags(e, st, cudaEventRecordExternal) : cudaEventRecord(e, st);
}
int index_ws(b200_index* idx, int slot, size_t bytes, void** out);
// Row scan + top-k of nq queries against rows [0, n) of `rows` (row-major fp16, d columns).
// Writes, per query, k sorted keys (local row ids) into d_keys_out [nq, k].
int scan_topk_keys(b200_index* idx, const __half* rows, int64_t n, const float* d_q, int nq, int k,
                   unsigned long long* d_keys_out, cudaStream_t st);
}  // namespace b200
