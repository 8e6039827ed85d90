// C ABI of the search path: the index object that replaces the FAISS index behind
// KnnService.knn_search (reference clip_retrieval/clip_back.py:343-399; the FAISS calls are
// load_index :589-596 and index.search_and_reconstruct :362).
#include "index.cuh"
#include "topk.cuh"
#include <float.h>
#include <algorithm>
#include <cstdlib>
#include <new>

namespace b200 {

__global__ void f32_to_f16_kernel(const float* __restrict__ in, __half* __restrict__ out, int64_t count) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) out[i] = __float2half_rn(in[i]);
}

// Reconstruct: one warp per (query, rank); key 0 -> all-ones bits (what FAISS leaves).  Keys hold local ids;
// `id_to_slot` (IVF) maps them to the list-ordered store, flat indexes store rows in id order.
__global__ void gather_rows_from_keys_kernel(const __half* __restrict__ rows, int d,
                                             const unsigned long long* __restrict__ keys,
                                             const uint32_t* __restrict__ id_to_slot, int64_t count,
                                             float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t w = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w >= count) return;
  const unsigned long long key = keys[w];
  float* o = out + w * d;
  if (key == 0ull) {
    for (int j = lane; j < d; j += 32) o[j] = __uint_as_float(0xffffffffu);
  } else {
    uint32_t slot = key_id(key);
    if (id_to_slot) slot = id_to_slot[slot];
    const __half* r = rows + (int64_t)slot * d;
    for (int j = lane; j < d; j += 32) o[j] = __half2float(r[j]);
  }
}

__global__ void gather_rows_from_slots_kernel(const __half* __restrict__ rows, int d,
                                              const int64_t* __restrict__ ids, int64_t id_base, int64_t ntotal,
                                              const uint32_t* __restrict__ id_to_slot, int64_t count,
                                              float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t w = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w >= count) return;
  int64_t local = ids[w] - id_base;
  float* o = out + w * d;
  if (ids[w] < 0 || local < 0 || local >= ntotal) {
    for (int j = lane; j < d; j += 32) o[j] = __uint_as_float(0xffffffffu);
  } else {
    if (id_to_slot) local = id_to_slot[local];
    const __half* r = rows + local * d;
    for (int j = lane; j < d; j += 32) o[j] = __half2float(r[j]);
  }
}

// Merge G per-shard sorted candidate lists (score desc, global id asc) into one top-k per query.
struct Cand {
  uint32_t ord;
  int64_t id;
};
__device__ __forceinline__ bool cand_before(const Cand& a, const Cand& b) {
  return a.ord > b.ord || (a.ord == b.ord && a.id < b.id);
}
// Dg / Ig point at shard 0's [nq, k] arrays; shard g's arrays sit g * stride_d / g * stride_i BYTES further (so the
// merge reads either [G, nq, k] arrays or an all-gathered buffer of packed per-shard blocks in place).
__global__ void __launch_bounds__(1024)
merge_shards_kernel(const float* __restrict__ Dg, const int64_t* __restrict__ Ig, size_t stride_d, size_t stride_i, int G,
                    int nq, int k, int P, float* __restrict__ D, int64_t* __restrict__ I) {
  extern __shared__ unsigned char smem_raw[];
  uint32_t* ords = reinterpret_cast<uint32_t*>(smem_raw);
  int64_t* ids = reinterpret_cast<int64_t*>(smem_raw + (size_t)P * 4 + ((P & 1) ? 4 : 0));
  const int q = blockIdx.x;
  const int M = G * k;
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    uint32_t o = 0;
    int64_t id = INT64_MAX;
    if (i < M) {
      const int g = i / k, j = i % k;
      const int64_t src = (int64_t)q * k + j;
      const int64_t gid = reinterpret_cast<const int64_t*>(reinterpret_cast<const char*>(Ig) + (size_t)g * stride_i)[src];
      if (gid >= 0) {
        o = f32_to_ordered(reinterpret_cast<const float*>(reinterpret_cast<const char*>(Dg) + (size_t)g * stride_d)[src]);
        id = gid;
      }
    }
    ords[i] = o;
    ids[i] = id;
  }
  __syncthreads();
  for (int size = 2; size <= P; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = threadIdx.x; i < (P >> 1); i += blockDim.x) {
        const int lo = 2 * i - (i & (stride - 1));
        const int hi = lo + stride;
        const bool up = (lo & size) == 0;
        Cand a{ords[lo], ids[lo]}, b{ords[hi], ids[hi]};
        if (cand_before(b, a) == up) {
          ords[lo] = b.ord; ids[lo] = b.id;
          ords[hi] = a.ord; ids[hi] = a.id;
        }
      }
      __syncthreads();
    }
  }
  for (int j = threadIdx.x; j < k; j += blockDim.x) {
    const bool empty = ids[j] == INT64_MAX;
    D[(int64_t)q * k + j] = empty ? -FLT_MAX : ordered_to_f32(ords[j]);
    I[(int64_t)q * k + j] = empty ? -1 : ids[j];
  }
}

// out[i] = map[I[i]] (an index file's ids for insertion ids); -1 and ids outside the map stay -1.
__global__ void ids_map_kernel(const int64_t* __restrict__ I, int64_t n, const int64_t* __restrict__ map, int64_t nmap,
                               int64_t* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t v = I[i];
  out[i] = (v >= 0 && v < nmap) ? map[v] : -1;
}

static int ensure_capacity(b200_index* idx, int64_t need) {
  if (need <= idx->capacity) return B200_OK;
  int64_t cap = need;
  if (!idx->reserved && idx->capacity > 0) cap = std::max<int64_t>(need, idx->capacity + idx->capacity / 2);
  __half* nr = nullptr;
  B200_CUDA(cudaMalloc((void**)&nr, (size_t)cap * idx->d * sizeof(__half)));
  if (idx->rows) {
    if (idx->ntotal > 0)
      B200_CUDA(cudaMemcpy(nr, idx->rows, (size_t)idx->ntotal * idx->d * sizeof(__half), cudaMemcpyDeviceToDevice));
    B200_CUDA(cudaFree(idx->rows));
  }
  idx->rows = nr;
  idx->capacity = cap;
  return B200_OK;
}

static int search_device_impl(b200_index* idx, const float* d_q, int nq, int k, float* d_D, int64_t* d_I, float* d_R,
                              cudaStream_t st) {
  B200_CHECK(nq >= 0 && k >= 1, B200_ERR_INVALID, "search: bad nq=%d k=%d", nq, k);
  if (nq == 0) return B200_OK;
  B200_CHECK(d_q && d_D && d_I, B200_ERR_INVALID, "search: null buffer");
  B200_CHECK(((uintptr_t)d_q & 15) == 0, B200_ERR_INVALID, "search: query buffer must be 16-byte aligned");
  idx->ev_used = 0;
  idx->last_scan_launches = 0;
  void* ws = nullptr;
  B200_TRY(index_ws(idx, 1, (size_t)nq * k * 8, &ws));
  unsigned long long* keys = (unsigned long long*)ws;
  if (idx->pq_M > 0) {
    B200_CHECK(!d_R || !idx->pt_A || idx->pt_orthonormal, B200_ERR_UNSUPPORTED,
               "search_and_reconstruct: the pre-transform matrix is not orthonormal, so rows cannot be mapped back");
    if (idx->host) return ivfpq_stream_search(idx, d_q, nq, k, keys, d_D, d_I, d_R, st);
    B200_TRY(ivf_finalize(idx));
    B200_TRY(ivfpq_search_keys(idx, d_q, nq, k, keys, st));
  } else if (idx->nlist > 0) {
    B200_TRY(ivf_finalize(idx));
    B200_TRY(ivf_search_keys(idx, d_q, nq, k, keys, st));   // keys carry insertion ids, not slots
  } else {
    B200_TRY(scan_topk_keys(idx, idx->rows, idx->ntotal, d_q, nq, k, keys, st));
  }
  B200_TRY(decode_keys(keys, (int64_t)nq * k, idx->id_base, nullptr, d_D, d_I, st));
  if (d_R && idx->pq_M > 0) {
    B200_TRY(ivfpq_decode(idx, keys, nullptr, (int64_t)nq * k, d_R, st));
  } else if (d_R) {
    const int64_t count = (int64_t)nq * k;
    gather_rows_from_keys_kernel<<<(unsigned)((count + 7) / 8), 256, 0, st>>>(idx->rows, idx->d, keys,
                                                                               idx->id_to_slot, count, d_R);
    B200_LAUNCH_OK();
  }
  return B200_OK;
}

static int merge_launch(const float* d_Dg, const int64_t* d_Ig, size_t stride_d, size_t stride_i, int G, int nq, int k,
                        float* d_D, int64_t* d_I, cudaStream_t st) {
  int P = 2;
  while (P < G * k) P <<= 1;
  const size_t smem = (size_t)P * 4 + ((P & 1) ? 4 : 0) + (size_t)P * 8;
  B200_CHECK(smem <= 200 * 1024, B200_ERR_UNSUPPORTED, "merge: G*k=%d exceeds 16384 candidates per query", G * k);
  if (smem > 48 * 1024)
    B200_CUDA(cudaFuncSetAttribute(merge_shards_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  merge_shards_kernel<<<nq, 1024, smem, st>>>(d_Dg, d_Ig, stride_d, stride_i, G, nq, k, P, d_D, d_I);
  B200_LAUNCH_OK();
  return B200_OK;
}

// packed per-shard blocks [I int64 nq*k | D f32 nq*k | padding], `stride` bytes apart (sharded.cu, sharded.py)
int merge_packed_launch(const void* d_gathered, int G, size_t stride, int nq, int k, float* d_D, int64_t* d_I,
                        cudaStream_t st) {
  const char* base = (const char*)d_gathered;
  return merge_launch((const float*)(base + (size_t)nq * k * 8), (const int64_t*)base, stride, stride, G, nq, k, d_D, d_I, st);
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_index_create_flat(int d, int device, b200_index** out) {
  B200_CHECK(out != nullptr, B200_ERR_INVALID, "create_flat: null out");
  B200_CHECK(d > 0 && d % 8 == 0 && d <= 2048, B200_ERR_INVALID, "create_flat: d=%d must be a multiple of 8, <= 2048", d);
  int ndev = 0;
  B200_CUDA(cudaGetDeviceCount(&ndev));
  B200_CHECK(device >= 0 && device < ndev, B200_ERR_INVALID, "create_flat: device %d of %d", device, ndev);
  b200_index* idx = new (std::nothrow) b200_index();
  B200_CHECK(idx != nullptr, B200_ERR_OOM, "create_flat: host allocation failed");
  if (const char* e = getenv("B200_GRAPHS")) idx->use_graphs = atoi(e) != 0;
  idx->d = d;
  idx->d_in = d;
  idx->row_bytes = 2 * d;
  idx->device = device;
  idx->sms = sm_count(device);
  *out = idx;
  return B200_OK;
}

int b200_index_create_ivfflat(int d, int nlist, const float* h_centroids, int device, b200_index** out) {
  B200_CHECK(nlist >= 1 && h_centroids != nullptr, B200_ERR_INVALID, "create_ivfflat: bad nlist/centroids");
  B200_TRY(b200_index_create_flat(d, device, out));
  DeviceGuard g(device);
  int rc = ivf_create(*out, nlist, h_centroids);
  if (rc != B200_OK) {
    b200_index_destroy(*out);
    *out = nullptr;
  }
  return rc;
}

int b200_index_destroy(b200_index* idx) {
  if (!idx) return B200_OK;
  DeviceGuard g(idx->device);
  cudaDeviceSynchronize();
  if (idx->rows) cudaFree(idx->rows);
  for (void* w : idx->ws)
    if (w) cudaFree(w);
  for (float* b : idx->norm_bound)
    if (b) cudaFree(b);
  for (auto e : idx->ev) cudaEventDestroy(e);
  for (auto& kv : idx->graphs) if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
  if (idx->cap_stream) cudaStreamDestroy(idx->cap_stream);
  if (idx->g_q) cudaFree(idx->g_q);
  if (idx->g_D) cudaFree(idx->g_D);
  if (idx->g_I) cudaFree(idx->g_I);
  if (idx->g_R) cudaFree(idx->g_R);
  ivf_free(idx);
  delete idx;
  return B200_OK;
}

int b200_index_reserve(b200_index* idx, int64_t n) {
  B200_CHECK(idx && n >= 0, B200_ERR_INVALID, "reserve: bad argument");
  DeviceGuard g(idx->device);
  idx->reserved = true;
  idx->graph_epoch++;
  if (idx->nlist > 0) return B200_OK;  // IVF sizes its store at finalize
  return ensure_capacity(idx, n);
}

static int add_rows(b200_index* idx, const void* rows, int64_t n, int on_device, bool f32) {
  B200_CHECK(idx && (rows || n == 0) && n >= 0, B200_ERR_INVALID, "add: bad argument");
  B200_CHECK(idx->pq_M == 0, B200_ERR_UNSUPPORTED,
             "add: an IVF-PQ index takes PQ codes (b200_index_add_codes); there is no encoder for float rows");
  if (n == 0) return B200_OK;
  idx->graph_epoch++;
  DeviceGuard g(idx->device);
  const int d = idx->d;
  __half* dst;
  if (idx->nlist > 0) {
    // IVF: stage in insertion order until finalize buckets them
    B200_TRY(grow_pending(idx, idx->npending + n, false));
    dst = idx->pending + idx->npending * d;
  } else {
    B200_CHECK(idx->ntotal + n < (1ll << 32), B200_ERR_UNSUPPORTED, "add: a shard holds at most 2^32 rows");
    B200_TRY(ensure_capacity(idx, idx->ntotal + n));
    dst = idx->rows + idx->ntotal * d;
  }
  if (!f32) {
    B200_CUDA(cudaMemcpy(dst, rows, (size_t)n * d * 2, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
  } else {
    const int64_t chunk = std::min<int64_t>(n, (64ll << 20) / d);  // rows per staging chunk
    const float* src = (const float*)rows;
    void* stage = nullptr;
    if (!on_device) B200_TRY(index_ws(idx, 2, (size_t)chunk * d * 4, &stage));
    for (int64_t r = 0; r < n; r += chunk) {
      const int64_t m = std::min(chunk, n - r);
      const float* dsrc = src + r * d;
      if (!on_device) {
        B200_CUDA(cudaMemcpy(stage, src + r * d, (size_t)m * d * 4, cudaMemcpyHostToDevice));
        dsrc = (const float*)stage;
      }
      const int64_t count = m * d;
      f32_to_f16_kernel<<<(unsigned)((count + 255) / 256), 256>>>(dsrc, dst + r * d, count);
      B200_LAUNCH_OK();
    }
    B200_CUDA(cudaDeviceSynchronize());
  }
  if (idx->nlist > 0) idx->npending += n;
  else idx->ntotal += n;
  return B200_OK;
}

int b200_index_add_f16(b200_index* idx, const void* rows, int64_t n, int rows_on_device) {
  return add_rows(idx, rows, n, rows_on_device, false);
}
int b200_index_add_f32(b200_index* idx, const float* rows, int64_t n, int rows_on_device) {
  return add_rows(idx, rows, n, rows_on_device, true);
}

int b200_index_add_assigned_f16(b200_index* idx, const void* rows, int64_t n, int rows_on_device, const int32_t* h_lists) {
  B200_CHECK(idx && h_lists, B200_ERR_INVALID, "add_assigned: bad argument");
  B200_CHECK(idx->nlist > 0, B200_ERR_STATE, "add_assigned: not an IVF index");
  B200_CHECK(idx->pq_M == 0, B200_ERR_UNSUPPORTED,
             "add_assigned: an IVF-PQ index takes PQ codes (b200_index_add_codes); there is no encoder for float rows");
  for (int64_t i = 0; i < n; i++)
    B200_CHECK(h_lists[i] >= 0 && h_lists[i] < idx->nlist, B200_ERR_INVALID, "add_assigned: row %lld has list %d of %d",
               (long long)i, h_lists[i], idx->nlist);
  const int64_t before = idx->npending;
  B200_TRY(add_rows(idx, rows, n, rows_on_device, false));
  idx->pending_lists.resize((size_t)before, 0xFFFFFFFFu);
  for (int64_t i = 0; i < n; i++) idx->pending_lists.push_back((uint32_t)h_lists[i]);
  return B200_OK;
}

int b200_index_add_synthetic(b200_index* idx, int64_t n, int64_t row0, const b200_synth_spec* spec) {
  B200_CHECK(idx && spec && n >= 0, B200_ERR_INVALID, "add_synthetic: bad argument");
  B200_CHECK(idx->pq_M == 0, B200_ERR_UNSUPPORTED,
             "add_synthetic: an IVF-PQ index takes PQ codes (b200_index_add_codes); there is no encoder for float rows");
  if (n == 0) return B200_OK;
  idx->graph_epoch++;
  DeviceGuard g(idx->device);
  if (idx->nlist > 0) return ivf_add_synthetic(idx, n, row0, spec);
  B200_CHECK(idx->ntotal + n < (1ll << 32), B200_ERR_UNSUPPORTED, "add: a shard holds at most 2^32 rows");
  B200_TRY(ensure_capacity(idx, idx->ntotal + n));
  B200_TRY(synth_rows<__half>(idx->rows + idx->ntotal * idx->d, n, idx->d, row0, spec, 0));
  B200_CUDA(cudaDeviceSynchronize());
  idx->ntotal += n;
  return B200_OK;
}

int b200_index_finalize(b200_index* idx) {
  B200_CHECK(idx, B200_ERR_INVALID, "finalize: null index");
  if (idx->nlist == 0) return B200_OK;
  DeviceGuard g(idx->device);
  return ivf_finalize(idx);
}

int64_t b200_index_ntotal(const b200_index* idx) { return idx ? idx->ntotal + idx->npending : -1; }
int b200_index_d(const b200_index* idx) { return idx ? idx->d_in : -1; }
int b200_index_pq_m(const b200_index* idx) { return idx ? idx->pq_M : -1; }
int b200_index_nlist(const b200_index* idx) { return idx ? idx->nlist : -1; }

int b200_index_set_id_base(b200_index* idx, int64_t id_base) {
  B200_CHECK(idx, B200_ERR_INVALID, "set_id_base: null index");
  idx->graph_epoch++;
  idx->id_base = id_base;
  return B200_OK;
}

int b200_index_set_nprobe(b200_index* idx, int nprobe) {
  B200_CHECK(idx, B200_ERR_INVALID, "set_nprobe: null index");
  B200_CHECK(idx->nlist > 0, B200_ERR_STATE, "set_nprobe: not an IVF index");
  B200_CHECK(nprobe >= 1, B200_ERR_INVALID, "set_nprobe: nprobe=%d", nprobe);
  idx->nprobe = std::min(nprobe, idx->nlist);
  return B200_OK;
}
int b200_index_get_nprobe(const b200_index* idx) { return idx ? idx->nprobe : -1; }

int b200_index_set_tensor_scan(b200_index* idx, int on) {
  B200_CHECK(idx, B200_ERR_INVALID, "set_tensor_scan: null index");
  idx->graph_epoch++;
  idx->use_mma = (on & 1) != 0;
  idx->use_staged = (on & 4) == 0;  // bit 2 set: also disable the cp.async.bulk ring (A/B)
  idx->use_hi_only = (on & 8) == 0; // bit 3 set: always the hi/lo split mode (no approximate pass)
  return B200_OK;
}

int b200_index_last_hi_only_fallbacks(const b200_index* idx) { return idx ? idx->last_hi_only_fallbacks : -1; }

int b200_index_last_scan_plan(const b200_index* idx, int32_t* h_plan) {
  B200_CHECK(idx && h_plan, B200_ERR_INVALID, "last_scan_plan: null argument");
  for (int i = 0; i < 4; i++) h_plan[i] = idx->last_scan_plan[i];
  return B200_OK;
}

int b200_index_ivf_lists(b200_index* idx, int64_t* h_sizes, int64_t* h_ids) {
  B200_CHECK(idx && h_sizes, B200_ERR_INVALID, "ivf_lists: null argument");
  B200_CHECK(idx->nlist > 0, B200_ERR_STATE, "ivf_lists: not an IVF index");
  DeviceGuard g(idx->device);
  B200_TRY(ivf_finalize(idx));
  return ivf_lists(idx, h_sizes, h_ids);
}

// nq <= 4 through a replayed CUDA graph: returns 1 when the search was served from a graph, 0 when the caller must
// launch eagerly (first sighting of the shape, graphs disabled, stream already capturing), < 0 on error.
static int search_graph(b200_index* idx, const float* d_q, int nq, int k, float* d_D, int64_t* d_I, float* d_R,
                        cudaStream_t st) {
  constexpr int GRAPH_MAX_NQ = 4;
  const size_t r_bytes = d_R ? (size_t)nq * k * idx->d_in * 4 : 0;
  // lists in host memory: every pass waits on the host for its probes, which a graph cannot replay
  if (!idx->use_graphs || nq < 1 || nq > GRAPH_MAX_NQ || k > 2048 || r_bytes > (8u << 20) || idx->npending > 0 || idx->host)
    return 0;
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  B200_CUDA(cudaStreamIsCapturing(st, &cs));
  if (cs != cudaStreamCaptureStatusNone) return 0;
  const uint64_t key = (uint64_t)nq | ((uint64_t)k << 8) | ((uint64_t)(idx->nlist > 0 ? idx->nprobe : 0) << 24) | ((uint64_t)(d_R != nullptr) << 56);
  b200_index::SearchGraph& sg = idx->graphs[key];
  if (sg.epoch != idx->graph_epoch) {
    if (sg.exec) cudaGraphExecDestroy(sg.exec);
    sg = b200_index::SearchGraph();
    sg.epoch = idx->graph_epoch;
  }
  if (sg.seen < 1) { sg.seen++; return 0; }        // first call of a shape runs eagerly (workspaces, attributes, events)
  // fixed buffers
  const size_t qb = (size_t)GRAPH_MAX_NQ * idx->d_in * 4;
  if (idx->g_q_cap < qb) {
    if (idx->g_q) B200_CUDA(cudaFree(idx->g_q));
    B200_CUDA(cudaMalloc((void**)&idx->g_q, qb));
    idx->g_q_cap = qb;
    idx->graph_epoch++; sg.epoch = idx->graph_epoch; if (sg.exec) { cudaGraphExecDestroy(sg.exec); sg.exec = nullptr; }
  }
  if (idx->g_k_cap < (size_t)GRAPH_MAX_NQ * k) {
    if (idx->g_D) B200_CUDA(cudaFree(idx->g_D));
    if (idx->g_I) B200_CUDA(cudaFree(idx->g_I));
    B200_CUDA(cudaMalloc((void**)&idx->g_D, (size_t)GRAPH_MAX_NQ * k * 4));
    B200_CUDA(cudaMalloc((void**)&idx->g_I, (size_t)GRAPH_MAX_NQ * k * 8));
    idx->g_k_cap = (size_t)GRAPH_MAX_NQ * k;
    idx->graph_epoch++; sg.epoch = idx->graph_epoch; if (sg.exec) { cudaGraphExecDestroy(sg.exec); sg.exec = nullptr; }
  }
  if (r_bytes > idx->g_r_cap) {
    if (idx->g_R) B200_CUDA(cudaFree(idx->g_R));
    B200_CUDA(cudaMalloc((void**)&idx->g_R, r_bytes));
    idx->g_r_cap = r_bytes;
    idx->graph_epoch++; sg.epoch = idx->graph_epoch; if (sg.exec) { cudaGraphExecDestroy(sg.exec); sg.exec = nullptr; }
  }
  if (sg.exec == nullptr) {
    cudaGraph_t graph = nullptr;
    const long long l0 = g_launches.load();
    // captured on a private stream (the caller's may be the legacy default stream, which cannot capture); the
    // instantiated graph is launched on the caller's stream
    if (!idx->cap_stream) B200_CUDA(cudaStreamCreateWithFlags(&idx->cap_stream, cudaStreamNonBlocking));
    B200_CUDA(cudaStreamBeginCapture(idx->cap_stream, cudaStreamCaptureModeThreadLocal));
    idx->capturing = true;
    const int rc = search_device_impl(idx, idx->g_q, nq, k, idx->g_D, idx->g_I, d_R ? idx->g_R : nullptr, idx->cap_stream);
    idx->capturing = false;
    const cudaError_t ce = cudaStreamEndCapture(idx->cap_stream, &graph);
    if (rc != B200_OK || ce != cudaSuccess || graph == nullptr) {
      if (graph) cudaGraphDestroy(graph);
      cudaGetLastError();
      idx->use_graphs = false;
      return rc != B200_OK ? rc : 0;
    }
    const cudaError_t ie = cudaGraphInstantiate(&sg.exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ie != cudaSuccess) { cudaGetLastError(); sg.exec = nullptr; idx->use_graphs = false; return 0; }
    sg.kernels = (int)(g_launches.load() - l0);
  }
  B200_CUDA(cudaMemcpyAsync(idx->g_q, d_q, (size_t)nq * idx->d_in * 4, cudaMemcpyDeviceToDevice, st));
  B200_CUDA(cudaGraphLaunch(sg.exec, st));
  B200_CUDA(cudaMemcpyAsync(d_D, idx->g_D, (size_t)nq * k * 4, cudaMemcpyDeviceToDevice, st));
  B200_CUDA(cudaMemcpyAsync(d_I, idx->g_I, (size_t)nq * k * 8, cudaMemcpyDeviceToDevice, st));
  if (d_R) B200_CUDA(cudaMemcpyAsync(d_R, idx->g_R, r_bytes, cudaMemcpyDeviceToDevice, st));
  count_launch(sg.kernels);
  return 1;
}

int b200_index_search_device(b200_index* idx, const float* d_q, int nq, int k, float* d_D, int64_t* d_I, float* d_R,
                             void* stream) {
  B200_CHECK(idx, B200_ERR_INVALID, "search: null index");
  std::lock_guard<std::mutex> lock(idx->mu);
  DeviceGuard g(idx->device);
  B200_TRY(idx->scratch.acquire((cudaStream_t)stream));
  int rc = B200_OK;
  if (d_q && d_D && d_I && nq >= 1 && k >= 1 && ((uintptr_t)d_q & 15) == 0) {
    if (idx->nlist > 0) B200_TRY(ivf_finalize(idx));
    rc = search_graph(idx, d_q, nq, k, d_D, d_I, d_R, (cudaStream_t)stream);
  }
  if (rc == 0) rc = search_device_impl(idx, d_q, nq, k, d_D, d_I, d_R, (cudaStream_t)stream);
  else if (rc == 1) rc = B200_OK;
  B200_TRY(idx->scratch.release((cudaStream_t)stream));
  return rc;
}

int b200_index_search(b200_index* idx, const float* h_q, int nq, int k, float* h_D, int64_t* h_I, float* h_R) {
  B200_CHECK(idx, B200_ERR_INVALID, "search: null index");
  B200_CHECK(nq >= 0 && k >= 1, B200_ERR_INVALID, "search: bad nq=%d k=%d", nq, k);
  if (nq == 0) return B200_OK;
  B200_CHECK(h_q && h_D && h_I, B200_ERR_INVALID, "search: null buffer");
  std::lock_guard<std::mutex> lock(idx->mu);
  DeviceGuard g(idx->device);
  const size_t qb = (size_t)nq * idx->d_in * 4, db = (size_t)nq * k * 4, ib = (size_t)nq * k * 8;
  const size_t rb = h_R ? (size_t)nq * k * idx->d_in * 4 : 0;
  auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
  void* ws = nullptr;
  B200_TRY(index_ws(idx, 2, al(qb) + al(db) + al(ib) + al(rb), &ws));
  char* p = (char*)ws;
  float* d_q = (float*)p; p += al(qb);
  float* d_D = (float*)p; p += al(db);
  int64_t* d_I = (int64_t*)p; p += al(ib);
  float* d_R = h_R ? (float*)p : nullptr;
  B200_TRY(idx->scratch.acquire(0));
  B200_CUDA(cudaMemcpyAsync(d_q, h_q, qb, cudaMemcpyHostToDevice, 0));
  B200_TRY(search_device_impl(idx, d_q, nq, k, d_D, d_I, d_R, 0));   // legacy stream: never captured
  B200_TRY(idx->scratch.release(0));
  B200_CUDA(cudaMemcpyAsync(h_D, d_D, db, cudaMemcpyDeviceToHost, 0));
  B200_CUDA(cudaMemcpyAsync(h_I, d_I, ib, cudaMemcpyDeviceToHost, 0));
  if (h_R) B200_CUDA(cudaMemcpyAsync(h_R, d_R, rb, cudaMemcpyDeviceToHost, 0));
  B200_CUDA(cudaStreamSynchronize(0));
  return B200_OK;
}

int b200_index_range_search(b200_index* idx, const float* h_q, float thresh, int64_t cap, float* h_D, int64_t* h_I,
                            int64_t* h_count) {
  B200_CHECK(idx && h_q && h_count && cap >= 0 && (cap == 0 || (h_D && h_I)), B200_ERR_INVALID, "range_search: bad argument");
  B200_CHECK(cap < (1ll << 31), B200_ERR_INVALID, "range_search: cap too large");
  std::lock_guard<std::mutex> lock(idx->mu);
  DeviceGuard g(idx->device);
  const size_t qb = ((size_t)idx->d_in * 4 + 255) & ~(size_t)255;
  void* ws = nullptr;
  B200_TRY(index_ws(idx, 2, qb + 256 + (size_t)cap * 8 + (size_t)cap * 12, &ws));
  float* d_q = (float*)ws;
  unsigned int* d_count = (unsigned int*)((char*)ws + qb);
  unsigned long long* d_keys = (unsigned long long*)((char*)ws + qb + 256);
  float* d_D = (float*)(d_keys + cap);
  int64_t* d_I = (int64_t*)((char*)d_D + (((size_t)cap * 4 + 7) & ~(size_t)7));
  B200_TRY(idx->scratch.acquire(0));
  B200_CUDA(cudaMemcpyAsync(d_q, h_q, (size_t)idx->d_in * 4, cudaMemcpyHostToDevice, 0));
  if (idx->host) {
    const int rc = ivfpq_stream_range(idx, d_q, thresh, d_keys, cap, d_count, h_D, h_I, h_count, 0);
    B200_TRY(idx->scratch.release(0));
    return rc;
  }
  if (idx->pq_M > 0) {
    B200_TRY(ivf_finalize(idx));
    B200_TRY(ivfpq_range_scan(idx, d_q, thresh, d_keys, (unsigned int)cap, d_count, 0));
  } else if (idx->nlist > 0) {
    B200_TRY(ivf_finalize(idx));
    B200_TRY(ivf_range_scan(idx, d_q, thresh, d_keys, (unsigned int)cap, d_count, 0));
  } else {
    B200_TRY(range_scan(idx, idx->rows, idx->ntotal, d_q, thresh, d_keys, (unsigned int)cap, d_count, 0));
  }
  unsigned int cnt = 0;
  B200_CUDA(cudaMemcpyAsync(&cnt, d_count, 4, cudaMemcpyDeviceToHost, 0));
  B200_CUDA(cudaStreamSynchronize(0));
  *h_count = cnt;
  const int64_t m = std::min<int64_t>(cnt, cap);
  if (m > 0) {
    B200_TRY(decode_keys(d_keys, m, idx->id_base, idx->nlist > 0 ? idx->row_ids : nullptr, d_D, d_I, 0));
    B200_CUDA(cudaMemcpyAsync(h_D, d_D, (size_t)m * 4, cudaMemcpyDeviceToHost, 0));
    B200_CUDA(cudaMemcpyAsync(h_I, d_I, (size_t)m * 8, cudaMemcpyDeviceToHost, 0));
    B200_CUDA(cudaStreamSynchronize(0));
  }
  return B200_OK;
}

int b200_index_reconstruct_device(b200_index* idx, const int64_t* d_ids, int64_t n, float* d_R, void* stream) {
  B200_CHECK(idx && d_ids && d_R && n >= 0, B200_ERR_INVALID, "reconstruct: bad argument");
  if (n == 0) return B200_OK;
  DeviceGuard g(idx->device);
  B200_CHECK(!idx->host, B200_ERR_UNSUPPORTED,
             "reconstruct: the lists are in host memory and the index keeps no id -> list map (FAISS's on-disk IVF "
             "without a direct map does not reconstruct either)");
  if (idx->pq_M > 0) {
    std::lock_guard<std::mutex> lock(idx->mu);
    B200_CHECK(!idx->pt_A || idx->pt_orthonormal, B200_ERR_UNSUPPORTED,
               "reconstruct: the pre-transform matrix is not orthonormal, so rows cannot be mapped back");
    B200_TRY(ivf_finalize(idx));
    return ivfpq_decode(idx, nullptr, d_ids, n, d_R, (cudaStream_t)stream);
  }
  const uint32_t* id_to_slot = nullptr;
  if (idx->nlist > 0) {
    std::lock_guard<std::mutex> lock(idx->mu);
    B200_TRY(ivf_finalize(idx));
    id_to_slot = idx->id_to_slot;
  }
  gather_rows_from_slots_kernel<<<(unsigned)((n + 7) / 8), 256, 0, (cudaStream_t)stream>>>(
      idx->rows, idx->d, d_ids, idx->id_base, idx->ntotal, id_to_slot, n, d_R);
  B200_LAUNCH_OK();
  return B200_OK;
}

int b200_ids_map_device(const int64_t* d_I, int64_t n, const int64_t* d_map, int64_t nmap, int64_t* d_out, int device,
                        void* stream) {
  B200_CHECK(d_I && d_map && d_out && n >= 0 && nmap >= 0, B200_ERR_INVALID, "ids_map: bad argument");
  if (n == 0) return B200_OK;
  DeviceGuard g(device);
  ids_map_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(d_I, n, d_map, nmap, d_out);
  B200_LAUNCH_OK();
  return B200_OK;
}

int b200_topk_merge_device(const float* d_Dg, const int64_t* d_Ig, int G, int nq, int k, float* d_D, int64_t* d_I,
                           int device, void* stream) {
  B200_CHECK(d_Dg && d_Ig && d_D && d_I && G >= 1 && nq >= 0 && k >= 1, B200_ERR_INVALID, "merge: bad argument");
  if (nq == 0) return B200_OK;
  DeviceGuard g(device);
  return merge_launch(d_Dg, d_Ig, (size_t)nq * k * 4, (size_t)nq * k * 8, G, nq, k, d_D, d_I, (cudaStream_t)stream);
}

int b200_topk_merge_packed_device(const void* d_gathered, int G, size_t shard_stride_bytes, int nq, int k, float* d_D,
                                  int64_t* d_I, int device, void* stream) {
  B200_CHECK(d_gathered && d_D && d_I && G >= 1 && nq >= 0 && k >= 1, B200_ERR_INVALID, "merge_packed: bad argument");
  B200_CHECK(shard_stride_bytes >= (size_t)nq * k * 12 && shard_stride_bytes % 8 == 0, B200_ERR_INVALID,
             "merge_packed: shard stride %zu too small for nq=%d k=%d or not a multiple of 8", shard_stride_bytes, nq, k);
  if (nq == 0) return B200_OK;
  DeviceGuard g(device);
  return merge_packed_launch(d_gathered, G, shard_stride_bytes, nq, k, d_D, d_I, (cudaStream_t)stream);
}

int b200_index_last_scan_ms(const b200_index* idx, float* ms, int* launches) {
  B200_CHECK(idx && ms, B200_ERR_INVALID, "last_scan_ms: null argument");
  DeviceGuard g(idx->device);
  float total = 0.f;
  for (int i = 0; i + 1 < idx->ev_used; i += 2) {
    B200_CUDA(cudaEventSynchronize(idx->ev[i + 1]));
    float t = 0.f;
    B200_CUDA(cudaEventElapsedTime(&t, idx->ev[i], idx->ev[i + 1]));
    total += t;
  }
  *ms = total;
  if (launches) *launches = idx->last_scan_launches;
  return B200_OK;
}

}  // extern "C"
