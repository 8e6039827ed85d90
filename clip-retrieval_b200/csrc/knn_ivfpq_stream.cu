// IVF-PQ with its lists in host memory: the on-disk index (`populated.index` + `merged_index.ivfdata`) served from
// the caller's read-only memory map, for collections whose codes do not fit in HBM.  Centroids, codebook and
// pre-transform stay on the device as for a resident index (knn_ivfpq.cu); the lists do not.  A search:
//   A. coarse step of every query on the GPU (pq_prepare), the probes [nq, nprobe] copied to the host;
//   B. passes: the host takes queries in order while the union of their probed lists fits the arena, numbers those
//      lists in ascending list id (arena list i), gathers their code rows from the map into pinned staging at the
//      store's pitch, and rewrites each probe key's list id into its arena list; a copy stream moves staging, arena
//      offsets and probes to the device; the compute stream waits for that copy, builds the tables, scans with
//      ivfpq_scan_kernel (row_ids = null: a key's id is its arena row), selects, and for search_and_reconstruct
//      decodes from the arena.  Two arenas: the host gathers pass p + 1 while the GPU copies and scans pass p.
//   C. the k keys of each query leave the GPU; the host maps arena row -> (arena list, position) -> the list's int64
//      id in the map.  Only kept rows' ids are read: ids never cross PCIe in bulk.
// Tie order: the arena holds a pass's lists in ascending list id with each list in file order, so arena rows of a
// query ascend with list-order slots, and a file loaded resident in list order gets insertion id = slot.  Equal
// scores therefore rank as in the resident load of the same file, and every output is the same bits.
#include "index.cuh"
#include <float.h>
#include <algorithm>
#include <chrono>
#include <cstring>
#include <thread>

namespace b200 {

constexpr size_t STREAM_ARENA_DEFAULT = 256u << 20;  // bytes per arena unless b200_index_set_stream_arena says otherwise

struct StreamBuf {
  uint8_t* d_arena = nullptr;
  uint8_t* h_stage = nullptr;                 // pinned [arena_rows, pitch]; padding bytes stay zero
  int64_t* h_off = nullptr;                   // pinned [nlist + 1]: arena row offsets of the pass's lists
  int64_t* d_off = nullptr;
  int32_t* h_lid = nullptr;                   // pinned [nlist]: arena list -> list id
  int32_t* d_lid = nullptr;
  unsigned long long* h_probes = nullptr;     // pinned [PQ_QB, nprobe]: probe keys naming arena lists
  unsigned long long* d_probes = nullptr;
  unsigned long long* h_keys = nullptr;       // pinned [PQ_QB, k]: the pass's selected keys
  cudaEvent_t copy_beg = nullptr, copy_end = nullptr, done = nullptr;
  int q0 = 0, qb = 0, nl = 0;                 // the pass it holds
  bool pending = false;
};

struct HostLists {
  std::vector<int64_t> sizes, starts;         // starts: list-order slot of each list's first row
  std::vector<const uint8_t*> codes;
  std::vector<const int64_t*> ids;
  size_t arena_bytes = STREAM_ARENA_DEFAULT;
  int64_t arena_rows = 0;                     // rows each arena holds (allocated)
  size_t probe_cap = 0, key_cap = 0;
  StreamBuf buf[2];
  cudaStream_t copy_st = nullptr;
  std::vector<int32_t> arena_of;              // list -> arena list of the pass being planned, -1 = not in it
  std::vector<int32_t> pass_lists;
  std::vector<unsigned long long> probes;     // [nq, nprobe] of the current search
  std::vector<float> out_D;
  std::vector<int64_t> out_I;
  double gather_ms = 0, copy_ms = 0;
  int64_t staged_bytes = 0;
  int passes = 0;
};

static float host_key_score(unsigned long long key) {   // ordered_to_f32 of common.cuh
  const uint32_t o = (uint32_t)(key >> 32);
  const uint32_t u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
static uint32_t host_key_id(unsigned long long key) { return ~(uint32_t)key; }

static void free_buf(StreamBuf& b) {
  if (b.d_arena) cudaFree(b.d_arena);
  if (b.h_stage) cudaFreeHost(b.h_stage);
  if (b.h_off) cudaFreeHost(b.h_off);
  if (b.d_off) cudaFree(b.d_off);
  if (b.h_lid) cudaFreeHost(b.h_lid);
  if (b.d_lid) cudaFree(b.d_lid);
  if (b.h_probes) cudaFreeHost(b.h_probes);
  if (b.d_probes) cudaFree(b.d_probes);
  if (b.h_keys) cudaFreeHost(b.h_keys);
  for (cudaEvent_t e : {b.copy_beg, b.copy_end, b.done})
    if (e) cudaEventDestroy(e);
  b = StreamBuf();
}

void host_lists_free(b200_index* idx) {
  if (!idx->host) return;
  for (StreamBuf& b : idx->host->buf) free_buf(b);
  if (idx->host->copy_st) cudaStreamDestroy(idx->host->copy_st);
  delete idx->host;
  idx->host = nullptr;
}

// Frees the device (or pinned) buffer *p and clears the pointer, then allocates `bytes` of it unless 0: a failed call
// leaves null, never a freed address.
template <typename T>
static int regrow(T** p, size_t bytes, bool pinned) {
  const cudaError_t e = *p ? (pinned ? cudaFreeHost(*p) : cudaFree(*p)) : cudaSuccess;
  *p = nullptr;
  B200_CUDA(e);
  if (bytes) B200_CUDA(pinned ? cudaHostAlloc((void**)p, bytes, cudaHostAllocDefault) : cudaMalloc((void**)p, bytes));
  return B200_OK;
}

// Arenas of max(arena_bytes / pitch, nprobe x the largest list) rows, so that one query always fits; probe and key
// staging for a pass of PQ_QB queries.
static int ensure_bufs(b200_index* idx, int nprobe, int k) {
  HostLists* H = idx->host;
  const int64_t pitch = idx->row_bytes;
  const int64_t rows = std::max<int64_t>({(int64_t)(H->arena_bytes / (size_t)pitch), (int64_t)nprobe * idx->max_list, 1});
  const size_t pcap = (size_t)PQ_QB * nprobe, kcap = (size_t)PQ_QB * k;
  if (!H->copy_st) B200_CUDA(cudaStreamCreateWithFlags(&H->copy_st, cudaStreamNonBlocking));
  for (StreamBuf& b : H->buf) {
    if (!b.done) {
      B200_CUDA(cudaEventCreate(&b.copy_beg));
      B200_CUDA(cudaEventCreate(&b.copy_end));
      B200_CUDA(cudaEventCreateWithFlags(&b.done, cudaEventDisableTiming));
      B200_CUDA(cudaHostAlloc((void**)&b.h_off, (size_t)(idx->nlist + 1) * 8, cudaHostAllocDefault));
      B200_CUDA(cudaMalloc((void**)&b.d_off, (size_t)(idx->nlist + 1) * 8));
      B200_CUDA(cudaHostAlloc((void**)&b.h_lid, (size_t)idx->nlist * 4, cudaHostAllocDefault));
      B200_CUDA(cudaMalloc((void**)&b.d_lid, (size_t)idx->nlist * 4));
    }
    if (rows > H->arena_rows) {
      B200_TRY(regrow(&b.d_arena, (size_t)rows * pitch, false));
      B200_TRY(regrow(&b.h_stage, (size_t)rows * pitch, true));
      memset(b.h_stage, 0, (size_t)rows * pitch);
    }
    if (pcap > H->probe_cap) {
      B200_TRY(regrow(&b.h_probes, pcap * 8, true));
      B200_TRY(regrow(&b.d_probes, pcap * 8, false));
    }
    if (kcap > H->key_cap) B200_TRY(regrow(&b.h_keys, kcap * 8, true));
  }
  H->arena_rows = std::max(H->arena_rows, rows);
  H->probe_cap = std::max(H->probe_cap, pcap);
  H->key_cap = std::max(H->key_cap, kcap);
  return B200_OK;
}

// Queries [a, *b) whose probed lists together fit the arena (at least query a; at most PQ_QB): their lists in
// ascending id become the arena lists of `B` (offsets, list ids), and their probe keys name arena lists.
static int plan_pass(b200_index* idx, StreamBuf& B, int nprobe, int a, int nq, int* b, int64_t* rows_out) {
  HostLists* H = idx->host;
  std::vector<int32_t>& L = H->pass_lists;
  L.clear();
  int64_t rows = 0;
  int q = a;
  for (; q < nq && q - a < PQ_QB; q++) {
    const size_t mark0 = L.size();
    int64_t add = 0;
    for (int p = 0; p < nprobe; p++) {
      const unsigned long long key = H->probes[(size_t)q * nprobe + p];
      if (key == 0ull) continue;
      const uint32_t l = host_key_id(key);
      if (H->arena_of[l] < 0) {
        H->arena_of[l] = 0;
        L.push_back((int32_t)l);
        add += H->sizes[l];
      }
    }
    if (rows + add > H->arena_rows && q > a) {
      for (size_t i = mark0; i < L.size(); i++) H->arena_of[L[i]] = -1;
      L.resize(mark0);
      break;
    }
    rows += add;
  }
  B200_CHECK(rows < (1ll << 32), B200_ERR_UNSUPPORTED,
             "search: a pass over lists in host memory holds at most 2^32 rows (%lld probed)", (long long)rows);
  std::sort(L.begin(), L.end());
  B.h_off[0] = 0;
  for (size_t i = 0; i < L.size(); i++) {
    H->arena_of[L[i]] = (int32_t)i;
    B.h_lid[i] = L[i];
    B.h_off[i + 1] = B.h_off[i] + H->sizes[L[i]];
  }
  for (int qq = a; qq < q; qq++)
    for (int p = 0; p < nprobe; p++) {
      const unsigned long long key = H->probes[(size_t)qq * nprobe + p];
      B.h_probes[(size_t)(qq - a) * nprobe + p] =
          key == 0ull ? 0ull : ((key & 0xffffffff00000000ull) | (uint32_t)~(uint32_t)H->arena_of[host_key_id(key)]);
    }
  for (int32_t l : L) H->arena_of[l] = -1;
  B.q0 = a;
  B.qb = q - a;
  B.nl = (int)L.size();
  *b = q;
  *rows_out = rows;
  return B200_OK;
}

// The code rows of B's arena lists from the map into pinned staging at the store's pitch: one copy per list when
// M fills the pitch (M % 16 == 0), else one per row.  A few host threads split the lists.
static void gather(b200_index* idx, StreamBuf& B, int64_t rows) {
  HostLists* H = idx->host;
  const int64_t pitch = idx->row_bytes, M = idx->pq_M;
  auto run = [&](int i0, int i1) {
    for (int i = i0; i < i1; i++) {
      const int32_t l = B.h_lid[i];
      const int64_t n = H->sizes[l];
      uint8_t* dst = B.h_stage + B.h_off[i] * pitch;
      const uint8_t* src = H->codes[l];
      if (pitch == M) {
        memcpy(dst, src, (size_t)n * M);
      } else {
        for (int64_t r = 0; r < n; r++) memcpy(dst + r * pitch, src + r * M, (size_t)M);
      }
    }
  };
  const int64_t bytes = rows * pitch;
  const int hw = (int)std::max(1u, std::thread::hardware_concurrency());
  const int T = bytes < (8ll << 20) ? 1 : std::min({8, hw, B.nl});
  if (T <= 1) {
    run(0, B.nl);
    return;
  }
  std::vector<std::thread> th;
  int i0 = 0;
  for (int t = 0; t < T; t++) {   // split by rows: thread t takes the lists starting in its share of the rows
    const int64_t end_row = rows * (t + 1) / T;
    int i1 = i0;
    while (i1 < B.nl && (t == T - 1 || B.h_off[i1] < end_row)) i1++;
    if (i1 > i0) th.emplace_back(run, i0, i1);
    i0 = i1;
  }
  for (auto& x : th) x.join();
}

// Arena row r of B -> (the index's list, position in that list).
static std::pair<int32_t, int64_t> arena_row(const StreamBuf& B, int64_t r) {
  const int a = (int)(std::upper_bound(B.h_off, B.h_off + B.nl + 1, r) - B.h_off) - 1;
  return {B.h_lid[a], r - B.h_off[a]};
}

// Keys of a finished pass -> D and the lists' own ids (+ id_base).
static int finish_pass(b200_index* idx, StreamBuf& B, int k) {
  HostLists* H = idx->host;
  B200_CUDA(cudaEventSynchronize(B.done));
  float ms = 0.f;
  B200_CUDA(cudaEventElapsedTime(&ms, B.copy_beg, B.copy_end));
  H->copy_ms += ms;
  for (int64_t i = 0; i < (int64_t)B.qb * k; i++) {
    const unsigned long long key = B.h_keys[i];
    const int64_t o = (int64_t)B.q0 * k + i;
    if (key == 0ull) {
      H->out_D[o] = -FLT_MAX;
      H->out_I[o] = -1;
      continue;
    }
    const auto [l, pos] = arena_row(B, host_key_id(key));
    H->out_D[o] = host_key_score(key);
    H->out_I[o] = idx->id_base + H->ids[l][pos];
  }
  B.pending = false;
  return B200_OK;
}

// Gather B's lists (timed), then enqueue the copy of staging, offsets, list ids and probe keys; copy_end follows all
// of them.
static int stage_pass(b200_index* idx, StreamBuf& B, int64_t rows, int nprobe, cudaStream_t cst) {
  HostLists* H = idx->host;
  const auto t0 = std::chrono::steady_clock::now();
  gather(idx, B, rows);
  H->gather_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  H->staged_bytes += rows * idx->row_bytes;
  H->passes++;
  B200_CUDA(cudaEventRecord(B.copy_beg, cst));
  if (rows > 0)
    B200_CUDA(cudaMemcpyAsync(B.d_arena, B.h_stage, (size_t)rows * idx->row_bytes, cudaMemcpyHostToDevice, cst));
  B200_CUDA(cudaMemcpyAsync(B.d_off, B.h_off, (size_t)(B.nl + 1) * 8, cudaMemcpyHostToDevice, cst));
  if (B.nl > 0) B200_CUDA(cudaMemcpyAsync(B.d_lid, B.h_lid, (size_t)B.nl * 4, cudaMemcpyHostToDevice, cst));
  B200_CUDA(cudaMemcpyAsync(B.d_probes, B.h_probes, (size_t)B.qb * nprobe * 8, cudaMemcpyHostToDevice, cst));
  B200_CUDA(cudaEventRecord(B.copy_end, cst));
  return B200_OK;
}

// Step A: probes of queries [0, nq) into H->probes.
static int all_probes(b200_index* idx, const PqSearch& s, const float* d_q, int nq, cudaStream_t st) {
  HostLists* H = idx->host;
  H->probes.resize((size_t)nq * s.nprobe);
  for (int b0 = 0; b0 < nq; b0 += PQ_QB) {
    const int bq = std::min(PQ_QB, nq - b0);
    B200_TRY(pq_prepare(idx, s, d_q + (size_t)b0 * idx->d_in, bq, true, nullptr, st));
    B200_CUDA(cudaMemcpyAsync(H->probes.data() + (size_t)b0 * s.nprobe, s.probes, (size_t)bq * s.nprobe * 8,
                              cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
  }
  return B200_OK;
}

static void reset_stats(HostLists* H) {
  H->gather_ms = H->copy_ms = 0;
  H->staged_bytes = 0;
  H->passes = 0;
}

int ivfpq_stream_search(b200_index* idx, const float* d_q, int nq, int k, unsigned long long* d_keys, float* d_D,
                        int64_t* d_I, float* d_R, cudaStream_t st) {
  HostLists* H = idx->host;
  PqSearch s;
  B200_TRY(pq_search_plan(idx, nq, k, &s));
  B200_TRY(ensure_bufs(idx, s.nprobe, k));
  reset_stats(H);
  H->out_D.resize((size_t)nq * k);
  H->out_I.resize((size_t)nq * k);
  B200_TRY(all_probes(idx, s, d_q, nq, st));
  int p = 0;
  for (int a = 0; a < nq; p++) {
    StreamBuf& B = H->buf[p & 1];
    if (B.pending) B200_TRY(finish_pass(idx, B, k));   // pass p - 2: its arena and staging are free again
    int b = a;
    int64_t rows = 0;
    B200_TRY(plan_pass(idx, B, s.nprobe, a, nq, &b, &rows));
    B200_TRY(stage_pass(idx, B, rows, s.nprobe, H->copy_st));
    float* tables = nullptr;
    B200_TRY(pq_prepare(idx, s, d_q + (size_t)a * idx->d_in, B.qb, false, &tables, st));
    B200_CUDA(cudaStreamWaitEvent(st, B.copy_end, 0));
    unsigned long long* keys = d_keys + (size_t)a * k;
    B200_TRY(pq_scan_select(idx, s, PqStore{B.d_arena, nullptr, B.d_off}, B.qb, tables, B.d_probes, keys, st));
    if (d_R)
      B200_TRY(pq_decode_launch(idx, B.d_arena, B.d_off, B.nl, B.d_lid, nullptr, keys, nullptr, (int64_t)B.qb * k,
                                d_R + (size_t)a * k * idx->d_in, st));
    B200_CUDA(cudaMemcpyAsync(B.h_keys, keys, (size_t)B.qb * k * 8, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaEventRecord(B.done, st));
    B.pending = true;
    a = b;
  }
  for (int i = 0; i < 2; i++) {   // the older pending pass first
    StreamBuf& B = H->buf[(p + i) & 1];
    if (B.pending) B200_TRY(finish_pass(idx, B, k));
  }
  B200_CUDA(cudaMemcpyAsync(d_D, H->out_D.data(), (size_t)nq * k * 4, cudaMemcpyHostToDevice, st));
  B200_CUDA(cudaMemcpyAsync(d_I, H->out_I.data(), (size_t)nq * k * 8, cudaMemcpyHostToDevice, st));
  B200_CUDA(cudaStreamSynchronize(st));
  return B200_OK;
}

int ivfpq_stream_range(b200_index* idx, const float* d_q, float thresh, unsigned long long* d_keys, int64_t cap,
                       unsigned int* d_count, float* h_D, int64_t* h_I, int64_t* h_count, cudaStream_t st) {
  HostLists* H = idx->host;
  PqSearch s;
  B200_TRY(pq_search_plan(idx, 1, 0, &s));
  B200_TRY(ensure_bufs(idx, s.nprobe, 1));
  reset_stats(H);
  B200_TRY(all_probes(idx, s, d_q, 1, st));
  StreamBuf& B = H->buf[0];
  int b = 0;
  int64_t rows = 0;
  B200_TRY(plan_pass(idx, B, s.nprobe, 0, 1, &b, &rows));
  B200_TRY(stage_pass(idx, B, rows, s.nprobe, st));
  float* tables = nullptr;
  B200_TRY(pq_prepare(idx, s, d_q, 1, false, &tables, st));
  B200_TRY(pq_scan_range(idx, s, PqStore{B.d_arena, nullptr, B.d_off}, tables, B.d_probes, thresh, d_keys,
                         (unsigned int)cap, d_count, st));
  unsigned int cnt = 0;
  B200_CUDA(cudaMemcpyAsync(&cnt, d_count, 4, cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  float ms = 0.f;
  B200_CUDA(cudaEventElapsedTime(&ms, B.copy_beg, B.copy_end));
  H->copy_ms += ms;
  *h_count = cnt;
  const int64_t m = std::min<int64_t>(cnt, cap);
  if (m == 0) return B200_OK;
  std::vector<unsigned long long> keys((size_t)m);
  B200_CUDA(cudaMemcpy(keys.data(), d_keys, (size_t)m * 8, cudaMemcpyDeviceToHost));
  // hits in ascending list-order slot: the order of the resident index's slot-keyed range search
  struct Hit { int64_t slot; float D; int64_t I; };
  std::vector<Hit> hits((size_t)m);
  for (int64_t i = 0; i < m; i++) {
    const auto [l, pos] = arena_row(B, host_key_id(keys[i]));
    hits[i] = Hit{H->starts[l] + pos, host_key_score(keys[i]), idx->id_base + H->ids[l][pos]};
  }
  std::sort(hits.begin(), hits.end(), [](const Hit& x, const Hit& y) { return x.slot < y.slot; });
  for (int64_t i = 0; i < m; i++) {
    h_D[i] = hits[i].D;
    h_I[i] = hits[i].I;
  }
  return B200_OK;
}

int ivfpq_stream_lists(b200_index* idx, int64_t* h_sizes, int64_t* h_ids) {
  HostLists* H = idx->host;
  for (int l = 0; l < idx->nlist; l++) h_sizes[l] = H->sizes[l];
  if (h_ids)
    for (int l = 0; l < idx->nlist; l++)
      for (int64_t i = 0; i < H->sizes[l]; i++) h_ids[H->starts[l] + i] = idx->id_base + H->ids[l][i];
  return B200_OK;
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_index_set_host_lists(b200_index* idx, int nlist, const int64_t* h_sizes, const uint64_t* h_code_addr,
                              const uint64_t* h_id_addr) {
  B200_CHECK(idx && h_sizes && h_code_addr && h_id_addr, B200_ERR_INVALID, "set_host_lists: null argument");
  B200_CHECK(idx->pq_M > 0, B200_ERR_STATE, "set_host_lists: not an IVF-PQ index");
  B200_CHECK(nlist == idx->nlist, B200_ERR_INVALID, "set_host_lists: %d lists for an index of nlist=%d", nlist, idx->nlist);
  std::lock_guard<std::mutex> lock(idx->mu);
  B200_CHECK(idx->host || (idx->ntotal == 0 && idx->npending == 0), B200_ERR_STATE,
             "set_host_lists: the index already holds %lld resident rows", (long long)(idx->ntotal + idx->npending));
  int64_t total = 0, max_list = 0;
  for (int l = 0; l < nlist; l++) {
    B200_CHECK(h_sizes[l] >= 0 && (h_sizes[l] == 0 || (h_code_addr[l] && h_id_addr[l])), B200_ERR_INVALID,
               "set_host_lists: list %d has size %lld and code / id addresses %#llx / %#llx", l, (long long)h_sizes[l],
               (unsigned long long)h_code_addr[l], (unsigned long long)h_id_addr[l]);
    total += h_sizes[l];
    max_list = std::max(max_list, h_sizes[l]);
  }
  DeviceGuard g(idx->device);
  if (!idx->host) idx->host = new HostLists();
  HostLists* H = idx->host;
  H->sizes.assign(h_sizes, h_sizes + nlist);
  H->starts.assign(nlist, 0);
  H->codes.resize(nlist);
  H->ids.resize(nlist);
  H->arena_of.assign(nlist, -1);
  for (int l = 0; l < nlist; l++) {
    H->starts[l] = l ? H->starts[l - 1] + h_sizes[l - 1] : 0;
    H->codes[l] = reinterpret_cast<const uint8_t*>((uintptr_t)h_code_addr[l]);
    H->ids[l] = reinterpret_cast<const int64_t*>((uintptr_t)h_id_addr[l]);
  }
  for (int l = 0; l <= nlist; l++) idx->h_list_offsets[l] = l < nlist ? H->starts[l] : total;
  idx->ntotal = total;
  idx->max_list = max_list;
  idx->graph_epoch++;
  return B200_OK;
}

int b200_index_set_stream_arena(b200_index* idx, size_t bytes) {
  B200_CHECK(idx, B200_ERR_INVALID, "set_stream_arena: null index");
  B200_CHECK(idx->host, B200_ERR_STATE, "set_stream_arena: the index has no lists in host memory (set_host_lists)");
  std::lock_guard<std::mutex> lock(idx->mu);
  DeviceGuard g(idx->device);
  idx->host->arena_bytes = bytes;
  // shrink: drop the arenas, the next search allocates what it needs
  idx->host->arena_rows = 0;
  for (StreamBuf& b : idx->host->buf) {
    B200_TRY(regrow(&b.d_arena, 0, false));
    B200_TRY(regrow(&b.h_stage, 0, true));
  }
  return B200_OK;
}

int b200_index_last_stream_stats(const b200_index* idx, double* h_stats) {
  B200_CHECK(idx && h_stats, B200_ERR_INVALID, "last_stream_stats: null argument");
  B200_CHECK(idx->host, B200_ERR_STATE, "last_stream_stats: the index has no lists in host memory");
  const HostLists* H = idx->host;
  h_stats[0] = H->gather_ms;
  h_stats[1] = H->copy_ms;
  h_stats[2] = (double)H->staged_bytes;
  h_stats[3] = H->passes;
  return B200_OK;
}

}  // extern "C"
