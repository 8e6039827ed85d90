// Shared helpers for the b200clip library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <string>
#include <atomic>
#include "../../include/b200clip.h"

namespace b200 {

// ---- error plumbing (no exception crosses the C ABI) -------------------------------------------
void set_error(const char* fmt, ...);
extern std::atomic<long long> g_launches;
inline void count_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

#define B200_CUDA(expr)                                                                      \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      ::b200::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__,   \
                        __LINE__);                                                           \
      return (_e == cudaErrorMemoryAllocation) ? B200_ERR_OOM : B200_ERR_CUDA;               \
    }                                                                                        \
  } while (0)

#define B200_CHECK(cond, code, ...)        \
  do {                                     \
    if (!(cond)) {                         \
      ::b200::set_error(__VA_ARGS__);      \
      return (code);                       \
    }                                      \
  } while (0)

#define B200_TRY(expr)          \
  do {                          \
    int _s = (expr);            \
    if (_s != B200_OK) return _s; \
  } while (0)

// Check the launch that was just issued.
#define B200_LAUNCH_OK()                                                                     \
  do {                                                                                       \
    ::b200::count_launch();                                                                  \
    cudaError_t _e = cudaGetLastError();                                                     \
    if (_e != cudaSuccess) {                                                                 \
      ::b200::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e),         \
                        __FILE__, __LINE__);                                                 \
      return B200_ERR_CUDA;                                                                  \
    }                                                                                        \
  } while (0)

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
    else prev = -1;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

int sm_count(int device);

// Buffers a handle shares between calls: calls hold the handle's mutex while they enqueue, acquire() before their
// first launch and release() after their last.  A call on a different stream than the previous one first waits (event)
// for the previous call's kernels, so in-flight work never sees its buffers reused.
struct StreamFence {
  cudaEvent_t ev = nullptr;   // recorded after the last call's launches
  cudaStream_t last = nullptr;
  bool used = false;
  ~StreamFence() {
    if (ev) cudaEventDestroy(ev);
  }
  int acquire(cudaStream_t st) {
    if (!ev) B200_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    if (used && last != st) B200_CUDA(cudaStreamWaitEvent(st, ev, 0));
    return B200_OK;
  }
  int release(cudaStream_t st) {
    B200_CUDA(cudaEventRecord(ev, st));
    last = st;
    used = true;
    return B200_OK;
  }
};

// ---- device helpers ---------------------------------------------------------------------------
__device__ __forceinline__ uint4 ld_nc_v4(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

// Total order on (score, id): higher score first, then lower id.  Packed so that a plain
// unsigned 64-bit compare implements it (larger key = better).  Key 0 is the empty-slot
// sentinel (decodes to id -1 / score -FLT_MAX); NaN scores are never turned into keys.
__device__ __forceinline__ uint32_t f32_to_ordered(float f) {
  uint32_t u = __float_as_uint(f + 0.0f);  // -0 -> +0
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ordered_to_f32(uint32_t o) {
  uint32_t u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
  return __uint_as_float(u);
}
__device__ __forceinline__ unsigned long long make_key(float score, uint32_t local_id) {
  return ((unsigned long long)f32_to_ordered(score) << 32) | (unsigned long long)(~local_id);
}
__device__ __forceinline__ float key_score(unsigned long long key) {
  return ordered_to_f32((uint32_t)(key >> 32));
}
__device__ __forceinline__ uint32_t key_id(unsigned long long key) { return ~(uint32_t)key; }

}  // namespace b200
