// Layer plumbing shared by the two encoder handles (clip_model.cu, text_encoder.cu): device allocations freed
// together, a GEMM layer with its weight maps, the attention over a fused qkv buffer, and per-class event timing.
#pragma once
#include "common.cuh"
#include "embed_kernels.cuh"
#include "gemm.cuh"
#include <algorithm>
#include <vector>

namespace b200 {

// Device allocations of a handle; its destroy frees them with free_all().
struct DeviceAllocs {
  std::vector<void*> ptrs;
  template <typename T>
  int alloc(T** p, size_t count) {
    void* q = nullptr;
    B200_CUDA(cudaMalloc(&q, std::max<size_t>(count, 1) * sizeof(T)));
    ptrs.push_back(q);
    *p = (T*)q;
    return B200_OK;
  }
  void free_all() {
    for (void* p : ptrs) cudaFree(p);
    ptrs.clear();
  }
};

struct Linear {
  __nv_bfloat16* w = nullptr;  // [N, K]
  float* b = nullptr;          // [N] or null
  int N = 0, K = 0;
  CUtensorMap tm128, tm64, tm32;   // weight boxes of BN rows x 64 columns for every tile width (256: two 128-row boxes)
};

// Zero-filled weight (and bias) of an N x K layer, with its tensor maps built once.
inline int make_linear(DeviceAllocs& allocs, Linear* l, int N, int K, bool bias) {
  l->N = N;
  l->K = K;
  B200_TRY(allocs.alloc(&l->w, (size_t)N * K));
  B200_CUDA(cudaMemset(l->w, 0, (size_t)N * K * 2));
  if (bias) {
    B200_TRY(allocs.alloc(&l->b, (size_t)N));
    B200_CUDA(cudaMemset(l->b, 0, (size_t)N * 4));
  }
  B200_TRY(make_tmap_2d(&l->tm128, l->w, 1, N, K, K, 128, GEMM_BK));
  B200_TRY(make_tmap_2d(&l->tm64, l->w, 1, N, K, K, 64, GEMM_BK));
  B200_TRY(make_tmap_2d(&l->tm32, l->w, 1, N, K, K, 32, GEMM_BK));
  return B200_OK;
}

// out = epilogue(A · l.w^T + l.b) at gemm_pick_bn's tile width; tmA has boxes of 128 rows x 64 columns.
inline int linear_gemm(const Linear& l, const CUtensorMap& tmA, int M, GemmEpilogue ep, int sms, cudaStream_t st) {
  const int bn = gemm_pick_bn(M, l.N, sms);
  ep.bias = l.b;
  const CUtensorMap& tmB = bn == 64 ? l.tm64 : (bn == 32 ? l.tm32 : l.tm128);
  return gemm_bf16_launch(tmA, tmB, bn, M, l.N, l.K, ep, st);
}

// qkv [planes, T, 3w] in boxes of 64 tokens x 64 columns: the Q / K / V tiles of the wgmma attention.
inline int make_qkv_map(CUtensorMap* tm, const __nv_bfloat16* qkv, int planes, int T, int w) {
  return make_tmap_3d(tm, qkv, 1, (uint64_t)planes, (uint64_t)T, 3 * (uint64_t)w, 3 * (uint64_t)w, (uint64_t)T * 3 * w,
                      64, 64);
}

// Attention over qkv [B*T, 3w] -> out [B*T, w]: the wgmma kernel where it applies, through `tm` (a make_qkv_map of at
// least B planes) or, when tm is null, a map built here; the mma.sync kernel otherwise.
inline int qkv_attention(const CUtensorMap* tm, const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int T, int heads,
                         int w, int causal, cudaStream_t st, const int* len = nullptr) {
  if (B > 0 && attention_wgmma_supported(T, heads, w)) {
    CUtensorMap own;
    if (tm == nullptr) {
      B200_TRY(make_qkv_map(&own, qkv, B, T, w));
      tm = &own;
    }
    return attention_wgmma(*tm, out, B, T, heads, w, causal, st, len);
  }
  return attention(qkv, out, B, T, heads, w, causal, st, len);
}

// Per-class device time of a handle's kernels: pairs of CUDA events around groups of launches, recorded only while
// profiling is on.  `launches` counts the kernels of every span, profiling or not.
struct SpanTimer {
  struct Span { int cls; cudaEvent_t a, b; };
  std::vector<Span> spans;   // events are reused across calls
  int used = 0;              // spans recorded since the last collect
  bool profiling = false;
  int launches = 0;
  ~SpanTimer() {
    for (auto& s : spans) { cudaEventDestroy(s.a); cudaEventDestroy(s.b); }
  }
  void set_profiling(bool on) {
    profiling = on;
    used = 0;
  }
  // ms[0 .. nclasses) = the summed time of each class's spans since the last collect; waits for them, then resets.
  int collect(float* ms, int nclasses) {
    for (int i = 0; i < nclasses; i++) ms[i] = 0.f;
    for (int i = 0; i < used; i++) {
      B200_CUDA(cudaEventSynchronize(spans[i].b));
      float t = 0.f;
      B200_CUDA(cudaEventElapsedTime(&t, spans[i].a, spans[i].b));
      if (spans[i].cls >= 0 && spans[i].cls < nclasses) ms[spans[i].cls] += t;
    }
    used = 0;
    return B200_OK;
  }
};

// The launches enqueued on `st` during its scope, as one span of class `cls` holding `kernels` kernels.
struct TimedSpan {
  SpanTimer& t;
  cudaStream_t st;
  int idx = -1;
  TimedSpan(SpanTimer& t_, int cls, cudaStream_t s, int kernels) : t(t_), st(s) {
    t.launches += kernels;
    if (!t.profiling) return;
    if (t.used == (int)t.spans.size()) {
      SpanTimer::Span sp;
      if (cudaEventCreate(&sp.a) != cudaSuccess || cudaEventCreate(&sp.b) != cudaSuccess) return;
      t.spans.push_back(sp);
    }
    idx = t.used++;
    t.spans[idx].cls = cls;
    cudaEventRecord(t.spans[idx].a, st);
  }
  ~TimedSpan() {
    if (idx >= 0) cudaEventRecord(t.spans[idx].b, st);
  }
};

}  // namespace b200
