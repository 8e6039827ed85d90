// Range-sharded search over the GPUs of one box behind the C ABI (SURVEY.md §8b `b200_sharded_search`, §8e):
// one host thread, one shard (b200_index) per device, queries replicated, local top-k with global ids, ONE
// exchange of the per-shard candidates, a device merge.  Two exchange modes:
//
//   comms == NULL  peer memory over NVLink/NVSwitch (the default): the last kernel of every shard's search
//                  (decode_keys, the top-k epilogue) stores its [nq, k] (id, score) block DIRECTLY into the
//                  root device's gathered buffer through a peer mapping — the "collective" is the epilogue's
//                  own stores; the root merges after one event wait per shard.  No NCCL launch, no pack/unpack.
//   comms != NULL  the NCCL protocol of the one-process-per-GPU deployment (sharded.py) inside one process:
//                  ncclAllGather of the packed blocks in one group, every device merges.  NCCL is resolved at
//                  run time (dlopen libnccl.so.2) so the library links without it.
//
// The reference has no sharded search (one CPU FAISS index per process, clip_back.py:781-782); the per-shard
// call is b200_index_search_device, the query API stays search(x, k) -> (D, I) (clip_back.py:362).
#include "index.cuh"
#include <dlfcn.h>
#include <mutex>
#include <algorithm>
#include <vector>

namespace b200 {

struct NcclApi {
  void* lib = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  int (*CommInitAll)(void**, int, const int*) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};

static NcclApi* nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);   // the copy already in the process (e.g. torch's)
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW);
    if (!h) return;
    api.lib = h;
    api.AllGather = (decltype(api.AllGather))dlsym(h, "ncclAllGather");
    api.GroupStart = (decltype(api.GroupStart))dlsym(h, "ncclGroupStart");
    api.GroupEnd = (decltype(api.GroupEnd))dlsym(h, "ncclGroupEnd");
    api.CommInitAll = (decltype(api.CommInitAll))dlsym(h, "ncclCommInitAll");
    api.CommDestroy = (decltype(api.CommDestroy))dlsym(h, "ncclCommDestroy");
    api.GetErrorString = (decltype(api.GetErrorString))dlsym(h, "ncclGetErrorString");
  });
  return (api.lib && api.AllGather && api.GroupStart && api.GroupEnd) ? &api : nullptr;
}

// per-root state of the sharded call (buffers on every device, streams, events); cached on the root index
struct ShardedState {
  int n = 0;
  std::vector<int> dev;
  std::vector<cudaStream_t> st;
  std::vector<cudaEvent_t> done;
  std::vector<float*> q;          // per device [nq, d]
  std::vector<char*> gathered;    // per device [G, block] (peer mode: root only)
  std::vector<float*> D;          // per device merged output
  std::vector<int64_t*> I;
  size_t q_cap = 0, block_cap = 0;
  bool peer_ok = false;
};

}  // namespace b200

using namespace b200;

struct b200_sharded {
  ShardedState s;
  std::vector<b200_index*> shards;
  std::mutex mu;
};

static void sharded_free_buffers(b200_sharded* h) {
  ShardedState& s = h->s;
  for (int i = 0; i < s.n; i++) {
    DeviceGuard g(s.dev[i]);
    if (s.q[i]) cudaFree(s.q[i]);
    if (s.gathered[i]) cudaFree(s.gathered[i]);
    if (s.D[i]) cudaFree(s.D[i]);
    if (s.I[i]) cudaFree(s.I[i]);
    s.q[i] = nullptr; s.gathered[i] = nullptr; s.D[i] = nullptr; s.I[i] = nullptr;
  }
  s.q_cap = s.block_cap = 0;
}

extern "C" {

int b200_sharded_create(b200_index* const* shards, int nshards, b200_sharded** out) {
  B200_CHECK(shards && out && nshards >= 1 && nshards <= 64, B200_ERR_INVALID, "sharded_create: bad argument");
  for (int i = 0; i < nshards; i++) {
    B200_CHECK(shards[i] != nullptr, B200_ERR_INVALID, "sharded_create: shard %d is null", i);
    B200_CHECK(shards[i]->d_in == shards[0]->d_in, B200_ERR_INVALID, "sharded_create: shard %d has d=%d, shard 0 has d=%d",
               i, shards[i]->d_in, shards[0]->d_in);
    for (int j = 0; j < i; j++)
      B200_CHECK(shards[j]->device != shards[i]->device, B200_ERR_INVALID,
                 "sharded_create: shards %d and %d share device %d (one shard per GPU)", j, i, shards[i]->device);
  }
  b200_sharded* h = new (std::nothrow) b200_sharded();
  B200_CHECK(h != nullptr, B200_ERR_OOM, "sharded_create: host allocation failed");
  ShardedState& s = h->s;
  s.n = nshards;
  h->shards.assign(shards, shards + nshards);
  s.dev.resize(nshards); s.st.assign(nshards, nullptr); s.done.assign(nshards, nullptr);
  s.q.assign(nshards, nullptr); s.gathered.assign(nshards, nullptr); s.D.assign(nshards, nullptr); s.I.assign(nshards, nullptr);
  for (int i = 0; i < nshards; i++) s.dev[i] = shards[i]->device;
  int rc = B200_OK;
  auto init = [&]() -> int {
    for (int i = 0; i < nshards; i++) {
      DeviceGuard g(s.dev[i]);
      B200_CUDA(cudaStreamCreateWithFlags(&s.st[i], cudaStreamNonBlocking));
      B200_CUDA(cudaEventCreateWithFlags(&s.done[i], cudaEventDisableTiming));
    }
    // peer mapping root <- every other shard (stores from device i into root memory)
    s.peer_ok = true;
    for (int i = 1; i < nshards; i++) {
      int can = 0;
      B200_CUDA(cudaDeviceCanAccessPeer(&can, s.dev[i], s.dev[0]));
      if (!can) { s.peer_ok = false; continue; }
      DeviceGuard g(s.dev[i]);
      cudaError_t e = cudaDeviceEnablePeerAccess(s.dev[0], 0);
      if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
      else if (e != cudaSuccess) { cudaGetLastError(); s.peer_ok = false; }
    }
    return B200_OK;
  };
  rc = init();
  if (rc != B200_OK) { b200_sharded_destroy(h); return rc; }
  *out = h;
  return B200_OK;
}

int b200_sharded_destroy(b200_sharded* h) {
  if (!h) return B200_OK;
  sharded_free_buffers(h);
  for (int i = 0; i < h->s.n; i++) {
    DeviceGuard g(h->s.dev[i]);
    if (h->s.st[i]) { cudaStreamSynchronize(h->s.st[i]); cudaStreamDestroy(h->s.st[i]); }
    if (h->s.done[i]) cudaEventDestroy(h->s.done[i]);
  }
  delete h;
  return B200_OK;
}

int b200_sharded_peer_mode(const b200_sharded* h) { return h ? (h->s.peer_ok ? 1 : 0) : -1; }

// index.search(x, k) over all shards: h_q fp32 [nq, d] host; h_D fp32 [nq, k]; h_I int64 [nq, k] (global ids).
// comms: NULL (peer-memory exchange; falls back to staged device-to-device copies when a pair of devices has no
// peer mapping) or an array of nshards ncclComm_t, comms[i] bound to shard i's device and rank i.
int b200_sharded_search(b200_sharded* h, void* const* comms, const float* h_q, int nq, int k, float* h_D, int64_t* h_I) {
  B200_CHECK(h && nq >= 0 && k >= 1, B200_ERR_INVALID, "sharded_search: bad argument");
  if (nq == 0) return B200_OK;
  B200_CHECK(h_q && h_D && h_I, B200_ERR_INVALID, "sharded_search: null buffer");
  std::lock_guard<std::mutex> lock(h->mu);
  ShardedState& s = h->s;
  const int G = s.n, d = h->shards[0]->d_in;   // query width
  const size_t q_bytes = (size_t)nq * d * 4;
  const size_t block = (((size_t)nq * k * 12) + 255) & ~(size_t)255;   // [I int64 nq*k | D f32 nq*k], padded
  NcclApi* nccl = nullptr;
  if (comms) {
    nccl = nccl_api();
    B200_CHECK(nccl != nullptr, B200_ERR_UNSUPPORTED, "sharded_search: libnccl.so.2 could not be loaded");
  }
  const bool all_gather_everywhere = comms != nullptr;
  if (q_bytes > s.q_cap || block > s.block_cap) {
    sharded_free_buffers(h);
    for (int i = 0; i < G; i++) {
      DeviceGuard g(s.dev[i]);
      B200_CUDA(cudaMalloc((void**)&s.q[i], q_bytes));
      B200_CUDA(cudaMalloc((void**)&s.gathered[i], (size_t)G * block));   // non-root: staging / NCCL receive buffer
      B200_CUDA(cudaMalloc((void**)&s.D[i], (size_t)nq * k * 4));
      B200_CUDA(cudaMalloc((void**)&s.I[i], (size_t)nq * k * 8));
    }
    s.q_cap = q_bytes;
    s.block_cap = block;
  }
  const size_t blk = s.block_cap;
  // 1. queries to every device, local search; the epilogue writes this shard's block
  for (int i = 0; i < G; i++) {
    DeviceGuard g(s.dev[i]);
    B200_CUDA(cudaMemcpyAsync(s.q[i], h_q, q_bytes, cudaMemcpyHostToDevice, s.st[i]));
    // where this shard's candidates land: its slot of the root's buffer (peer store) or of its own buffer
    const bool direct = !all_gather_everywhere && (i == 0 || s.peer_ok);
    char* slot = (direct ? s.gathered[0] : s.gathered[i]) + (size_t)i * blk;
    int64_t* dI = (int64_t*)slot;
    float* dD = (float*)(slot + (size_t)nq * k * 8);
    B200_TRY(b200_index_search_device(h->shards[i], s.q[i], nq, k, dD, dI, nullptr, s.st[i]));
    if (!all_gather_everywhere && !direct)   // no peer mapping: one explicit copy into the root's slot
      B200_CUDA(cudaMemcpyPeerAsync(s.gathered[0] + (size_t)i * blk, s.dev[0], slot, s.dev[i], blk, s.st[i]));
    B200_CUDA(cudaEventRecord(s.done[i], s.st[i]));
  }
  // 2. exchange + merge
  if (all_gather_everywhere) {
    int e = nccl->GroupStart();
    for (int i = 0; i < G && e == 0; i++) {
      DeviceGuard g(s.dev[i]);
      e = nccl->AllGather(s.gathered[i] + (size_t)i * blk, s.gathered[i], blk, /*ncclInt8*/ 0, comms[i], s.st[i]);
    }
    const int e2 = nccl->GroupEnd();
    if (e == 0) e = e2;
    B200_CHECK(e == 0, B200_ERR_CUDA, "sharded_search: NCCL all-gather failed: %s",
               nccl->GetErrorString ? nccl->GetErrorString(e) : "?");
    for (int i = 0; i < G; i++) {
      DeviceGuard g(s.dev[i]);
      B200_TRY(merge_packed_launch(s.gathered[i], G, blk, nq, k, s.D[i], s.I[i], s.st[i]));
    }
  } else {
    DeviceGuard g(s.dev[0]);
    for (int i = 1; i < G; i++) B200_CUDA(cudaStreamWaitEvent(s.st[0], s.done[i], 0));
    B200_TRY(merge_packed_launch(s.gathered[0], G, blk, nq, k, s.D[0], s.I[0], s.st[0]));
  }
  // 3. result of the root to the host
  {
    DeviceGuard g(s.dev[0]);
    B200_CUDA(cudaMemcpyAsync(h_D, s.D[0], (size_t)nq * k * 4, cudaMemcpyDeviceToHost, s.st[0]));
    B200_CUDA(cudaMemcpyAsync(h_I, s.I[0], (size_t)nq * k * 8, cudaMemcpyDeviceToHost, s.st[0]));
    B200_CUDA(cudaStreamSynchronize(s.st[0]));
  }
  if (all_gather_everywhere)
    for (int i = 1; i < G; i++) {
      DeviceGuard g(s.dev[i]);
      B200_CUDA(cudaStreamSynchronize(s.st[i]));
    }
  return B200_OK;
}

// Convenience for hosts without their own NCCL bootstrap (and for the tests): ncclCommInitAll over `devices`.
int b200_nccl_comm_init_all(int n, const int* devices, void** comms_out) {
  B200_CHECK(n >= 1 && devices && comms_out, B200_ERR_INVALID, "nccl_comm_init_all: bad argument");
  NcclApi* nccl = nccl_api();
  B200_CHECK(nccl != nullptr && nccl->CommInitAll, B200_ERR_UNSUPPORTED, "nccl_comm_init_all: libnccl.so.2 could not be loaded");
  const int e = nccl->CommInitAll(comms_out, n, devices);
  B200_CHECK(e == 0, B200_ERR_CUDA, "ncclCommInitAll failed: %s", nccl->GetErrorString ? nccl->GetErrorString(e) : "?");
  return B200_OK;
}
int b200_nccl_comm_destroy(void* comm) {
  NcclApi* nccl = nccl_api();
  B200_CHECK(nccl != nullptr && nccl->CommDestroy, B200_ERR_UNSUPPORTED, "nccl_comm_destroy: libnccl.so.2 could not be loaded");
  if (comm) nccl->CommDestroy(comm);
  return B200_OK;
}

}  // extern "C"
