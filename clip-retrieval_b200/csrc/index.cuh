// The index handle behind b200_index* (flat, IVF-Flat and IVF-PQ share the row store and the top-k tail).
#pragma once
#include "common.cuh"
#include <algorithm>
#include <map>
#include <mutex>
#include <vector>

namespace b200 { struct HostLists; }

struct b200_index {
  int d = 0;                // width of the stored space (IVF-PQ: the code space, after any pre-transform)
  int d_in = 0;             // width of a query and of a reconstructed row (== d unless a pre-transform is set)
  int row_bytes = 0;        // bytes per stored row: 2 * d (fp16 rows) or the 16-byte padded code pitch (IVF-PQ)
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
  uint32_t* id_to_slot = nullptr;         // device [ntotal]: inverse of row_ids, rebuilt whenever the store changes

  // IVF-PQ (8-bit codes): `rows` holds M code bytes per row at a pitch of row_bytes, list after list
  int pq_M = 0;                     // 0 = not IVF-PQ
  bool pq_by_residual = true;
  float* pq_centroids = nullptr;    // device [nlist, d] fp32 (dis0 and decoding; never the fp16 copy)
  float* pq_codebook = nullptr;     // device [M, 256, d / M] fp32
  float* pt_A = nullptr;            // device [d, d_in] fp32: q' = A q + b; null = no pre-transform
  float* pt_b = nullptr;            // device [d] fp32
  bool pt_orthonormal = false;      // rows of A orthonormal: reconstruct may apply A^T (y - b)
  // lists in host memory (b200_index_set_host_lists): `rows` stays empty, each query pass stages its probed lists
  // into a device arena (knn_ivfpq_stream.cu).  null = the resident store above.
  b200::HostLists* host = nullptr;

  // scratch
  void* ws[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // 0: scan internals; 1..3: callers; 4,5: hi-only mode
  size_t ws_bytes[6] = {0, 0, 0, 0, 0, 0};
  std::mutex mu;             // every search entry (host and device) holds it while it enqueues work
  b200::StreamFence scratch; // orders the searches that reuse ws[] / norm_bound[] / timing events across streams

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
  // {kernel, queries per pass, 16-byte chunks per lane, ring stages} of the last eager exhaustive scan;
  // kernel: 0 register FMA, 1 staged FMA (bulk-copy ring), 2 wgmma split, 3 wgmma hi-only.  -1 before any scan.
  // kernel 4: IVF-PQ list scan {4, sub-quantisers per CTA, CTAs per cluster, candidate warps per CTA}.
  int last_scan_plan[4] = {-1, -1, -1, -1};
};

namespace b200 {
inline cudaError_t index_record(b200_index* idx, cudaEvent_t e, cudaStream_t st) {
  return idx->capturing ? cudaEventRecordWithFlags(e, st, cudaEventRecordExternal) : cudaEventRecord(e, st);
}
// Scan timing: one event pair around the row-scan launches of a query batch (read by b200_index_last_scan_ms).
inline int scan_timer_begin(b200_index* idx, cudaStream_t st) {
  if ((int)idx->ev.size() < idx->ev_used + 2) {
    cudaEvent_t a, b;
    B200_CUDA(cudaEventCreate(&a));
    B200_CUDA(cudaEventCreate(&b));
    idx->ev.push_back(a);
    idx->ev.push_back(b);
  }
  B200_CUDA(index_record(idx, idx->ev[idx->ev_used], st));
  return B200_OK;
}
inline int scan_timer_end(b200_index* idx, cudaStream_t st) {
  B200_CUDA(index_record(idx, idx->ev[idx->ev_used + 1], st));
  idx->ev_used += 2;
  return B200_OK;
}

inline int next_pow2(int x) {
  int p = 1;
  while (p < x) p <<= 1;
  return p;
}

// Segments per probed list: enough CTAs over the `work_items` (query, probe) pairs of a launch to reach
// `target_ctas`, at most 32, and no segment shorter than about `min_rows` rows of the longest list.
inline int list_segments(const b200_index* idx, int target_ctas, int64_t work_items, int min_rows) {
  const int64_t segs = std::min<int64_t>(32, std::max<int64_t>(1, (target_ctas + work_items - 1) / work_items));
  return (int)std::max<int64_t>(1, std::min<int64_t>(segs, (idx->max_list + min_rows - 1) / min_rows));
}

// ---- knn_scan.cu ------------------------------------------------------------------------------------
int index_ws(b200_index* idx, int slot, size_t bytes, void** out);
// Row scan + top-k of nq queries against rows [0, n) of `rows` (row-major fp16, d columns).
// Writes, per query, k sorted keys (local row ids) into d_keys_out [nq, k].
int scan_topk_keys(b200_index* idx, const __half* rows, int64_t n, const float* d_q, int nq, int k,
                   unsigned long long* d_keys_out, cudaStream_t st);
// One query: appends up to `cap` keys to d_out, *d_count receives the number of hits (may exceed cap).
int range_scan(b200_index* idx, const __half* rows, int64_t n, const float* d_q, float thresh, unsigned long long* d_out,
               unsigned int cap, unsigned int* d_count, cudaStream_t st);
// keys -> (D, I): key 0 -> (-FLT_MAX, -1); `slot_to_id` (or null) maps the key's id before id_base is added.
int decode_keys(const unsigned long long* keys, int64_t count, int64_t id_base, const uint32_t* slot_to_id, float* D,
                int64_t* I, cudaStream_t st);

// The select tail of every search: M candidate keys per query -> the k best, sorted.  Level 1 cuts the candidates
// into `slices` chunks of about C keys and keeps k of each; level 2 merges the slices * k survivors in one block
// with a C2-entry buffer.
constexpr size_t SELECT_SMEM_MAX = 200 * 1024;   // shared memory of one select block; bounds C, hence k
inline int select_buffer(int k) { return std::max(2048, next_pow2(2 * k)); }   // C: entries of a block's sort buffer
struct SelectPlan {
  int64_t M = 0;
  int k = 0, C = 0, slices = 0, C2 = 0;
  size_t keys(int nq) const { return (size_t)nq * (M + (int64_t)slices * k); }   // scratch: candidates + level-1 output
};
// Fails with B200_ERR_UNSUPPORTED when k is beyond what one select block holds.
int plan_select(int64_t M, int k, SelectPlan* p);
// cand [nq, M] -> out [nq, k] through tmp [nq, slices * k]: two topk_select_kernel launches.
int select_topk(const SelectPlan& p, const unsigned long long* cand, unsigned long long* tmp, unsigned long long* out,
                int nq, cudaStream_t st);
// One launch of topk_select_kernel: grid (slices, nq), the k best of each slice of the M keys of a query.
int launch_topk_select(const unsigned long long* in, int64_t in_stride_q, int64_t M, int k, int C,
                       unsigned long long* out, int64_t out_stride_q, int slices, int nq, cudaStream_t st);

// ---- knn_mma.cu: batched scan on the tensor cores, same contract as scan_topk_keys ---------------------
int scan_topk_keys_mma(b200_index* idx, const __half* rows, int64_t n, const float* d_q, int nq, int k,
                       unsigned long long* d_keys_out, cudaStream_t st);

// ---- knn_ivf.cu ---------------------------------------------------------------------------------------
int ivf_create(b200_index* idx, int nlist, const float* h_centroids);
int ivf_finalize(b200_index* idx);
int ivf_add_synthetic(b200_index* idx, int64_t n, int64_t row0, const b200_synth_spec* spec);
int ivf_search_keys(b200_index* idx, const float* d_q, int nq, int k, unsigned long long* d_keys, cudaStream_t st);
int ivf_lists(b200_index* idx, int64_t* h_sizes, int64_t* h_ids);
void ivf_free(b200_index* idx);
// One query (device pointer): (score, slot) keys of every probed row above `thresh`; *d_count = number of hits.
int ivf_range_scan(b200_index* idx, const float* d_q, float thresh, unsigned long long* d_out, unsigned int cap,
                   unsigned int* d_count, cudaStream_t st);
// Room for `need` rows of row_bytes in idx->pending (contents kept).  `amortised`: grow by at least half the
// capacity, for callers that add a few rows at a time; otherwise exactly to `need`.
int grow_pending(b200_index* idx, int64_t need, bool amortised);

// ---- knn_ivfpq.cu ---------------------------------------------------------------------------------------
constexpr int PQ_QB = 256;   // queries per batch or streamed pass at most (bounds the tables scratch)
struct PqPlan {
  int cs = 0, mc = 0, warps = 0;
  size_t smem = 0;
};
// What a list scan reads: codes at the index's pitch list after list, list offsets [lists + 1], and the key id of each
// row (null: the row itself).  The resident store, or a staging arena of host-memory lists.
struct PqStore {
  const uint8_t* codes;
  const uint32_t* row_ids;
  const int64_t* offsets;
};
// Everything an IVF-PQ search decides before its first launch, whether its lists sit in HBM or in host memory: the
// coarse select `cp`, the list-scan plan `pl`, `segs` segments per probed list, `cpq` clusters per query, Mq candidates
// per query and their select `sel`, for batches of at most qmax queries; and the scratch: w0 the coarse scores and the
// candidates, `probes` [qmax, nprobe], w4 the code-space queries and the tables.
struct PqSearch {
  int nprobe = 0, k = 0, qmax = 0, segs = 0, cpq = 0;
  int64_t Mq = 0;
  SelectPlan cp, sel;
  PqPlan pl;
  unsigned long long* w0 = nullptr;
  unsigned long long* probes = nullptr;
  float* w4 = nullptr;
};
// Top-k search of nq queries; a range search plans one query with k = 0 (no candidates, an empty select).
int pq_search_plan(b200_index* idx, int nq, int k, PqSearch* s);
// Steps (0)-(2) for queries [0, qb) of d_q: the code-space queries, then when `probes` is set their probes into s.probes,
// then when `tables` is non-null their tables [qb, pitch, 256] into scratch at *tables.
int pq_prepare(b200_index* idx, const PqSearch& s, const float* d_q, int qb, bool probes, float** tables, cudaStream_t st);
// The list scan of qb queries' `probes` [qb, nprobe] over `store` (timed, counted, its plan recorded), then the select of
// each query's k best into out [qb, k].
int pq_scan_select(b200_index* idx, const PqSearch& s, const PqStore& store, int qb, const float* tables,
                   const unsigned long long* probes, unsigned long long* out, cudaStream_t st);
// The range scan of one query: *counter = 0, then every row above `thresh` appended to out (up to `cap` keys).
int pq_scan_range(b200_index* idx, const PqSearch& s, const PqStore& store, const float* tables,
                  const unsigned long long* probes, float thresh, unsigned long long* out, unsigned int cap,
                  unsigned int* counter, cudaStream_t st);
int pq_decode_launch(b200_index* idx, const uint8_t* codes, const int64_t* offsets, int nlists, const int32_t* list_ids,
                     const uint32_t* id_to_slot, const unsigned long long* keys, const int64_t* ids, int64_t count,
                     float* d_R, cudaStream_t st);
int ivfpq_search_keys(b200_index* idx, const float* d_q, int nq, int k, unsigned long long* d_keys, cudaStream_t st);
// One query (device pointer): (score, slot) keys of every row of the probed lists scoring strictly above `thresh`.
int ivfpq_range_scan(b200_index* idx, const float* d_q, float thresh, unsigned long long* d_out, unsigned int cap,
                     unsigned int* d_count, cudaStream_t st);
// Rows for keys (search_and_reconstruct) or for ids (reconstruct); exactly one of the two is non-null.
int ivfpq_decode(b200_index* idx, const unsigned long long* keys, const int64_t* ids, int64_t count, float* d_R,
                 cudaStream_t st);

// ---- knn_ivfpq_stream.cu: IVF-PQ with lists in host memory --------------------------------------------------------
// search: D, I (the lists' own ids + id_base) into device d_D / d_I, the decoded rows into d_R (or null), each pass
// decoding from its arena; d_keys [nq, k] is scratch.  Returns with the stream synchronised.
int ivfpq_stream_search(b200_index* idx, const float* d_q, int nq, int k, unsigned long long* d_keys, float* d_D,
                        int64_t* d_I, float* d_R, cudaStream_t st);
// range_search of one query (d_keys [cap] and d_count are scratch): up to `cap` hits into h_D / h_I in ascending
// list-order slot; *h_count = all hits.
int ivfpq_stream_range(b200_index* idx, const float* d_q, float thresh, unsigned long long* d_keys, int64_t cap,
                       unsigned int* d_count, float* h_D, int64_t* h_I, int64_t* h_count, cudaStream_t st);
int ivfpq_stream_lists(b200_index* idx, int64_t* h_sizes, int64_t* h_ids);
void host_lists_free(b200_index* idx);

// ---- pq_encode.cu: the PQ pieces OPQ training (opq_train.cu) reuses ---------------------------------------
// Y [n, d] = X [n, d_in] A^T (+ b): the row pre-transform of encode.
int pq_pretransform(const float* X, int64_t n, int d_in, const float* A, const float* b, int d, float* Y, cudaStream_t st);
// codes [n, M] of rows X [n, d] against the codebook (no residual).
int pq_codes(const float* X, int64_t n, int d, int M, const float* cb, uint8_t* codes, cudaStream_t st);
// Initial codebook [M, 256, d / M] of b200_pq_train_f32: sub-vectors of one seeded pick per stride of the rows.
int pq_init_codebook(const float* d_x, int64_t n, int d, int M, uint64_t seed, float* cb);
// The Lloyd iterations of b200_pq_train_f32, started from the device codebook `cb` (updated in place).
// codes_out (device [n, M] or null) receives the codes of the final codebook; h_sizes [M, 256] (or null) its sizes.
int pq_train_loop(const float* d_x, int64_t n, int d, int M, int niter, float* cb, uint8_t* codes_out, int64_t* h_sizes);

// ---- knn_index.cu -----------------------------------------------------------------------------------------
// packed per-shard blocks [I int64 nq*k | D f32 nq*k | padding], `stride` bytes apart (sharded.cu, sharded.py)
int merge_packed_launch(const void* d_gathered, int G, size_t stride, int nq, int k, float* d_D, int64_t* d_I,
                        cudaStream_t st);

// ---- synth.cu: deterministic synthetic rows (OutT = __half or float) -------------------------------------
template <typename OutT>
int synth_rows(OutT* d_out, int64_t n, int d, int64_t row0, const b200_synth_spec* spec, cudaStream_t st);
// out[p] = synthetic row (row0 + src_rows[p])
int synth_rows_indirect_f16(__half* out, const uint32_t* src_rows, int64_t n, int d, int64_t row0,
                            const b200_synth_spec* spec, cudaStream_t st);
}  // namespace b200
