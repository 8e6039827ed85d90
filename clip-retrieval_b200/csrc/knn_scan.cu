// Search path, exhaustive scan: the kernel behind index.search / search_and_reconstruct for the flat
// index (reference call site clip_retrieval/clip_back.py:362) and behind the coarse step of IVF.
//
// HBM-bound design (SURVEY.md §8d row 3, nq small): every fp16 row is read exactly once with
// 128-bit non-allocating loads, a warp owns U consecutive rows per step (U*d*2 bytes in flight per
// warp), fp32 FMA against up to NQ queries held in registers, one transposing shuffle reduction
// for the U*NQ dot products, and a per-warp replace-worst candidate list in shared memory that is
// touched only when a score beats the list's current worst (k*(1+ln(n_warp/k)) times per warp).
// Algorithmic bytes per launch: n * d * 2 (the row store); everything else is O(grid * k).
#include "index.cuh"
#include "scan.cuh"
#include <float.h>
#include <algorithm>

namespace b200 {

constexpr int SCAN_U = 4;

// After the transposing reduction of a block of SCAN_U rows x NQ queries starting at row r0: the lanes holding a
// total offer (score, row) to the list of their query.
template <int NQ>
__device__ __forceinline__ void offer_block_scores(float s, int64_t r0, int64_t n, int nq_valid, unsigned long long* wkeys,
                                                   int k, unsigned long long (&worst)[NQ], int (&worst_pos)[NQ], int lane) {
  constexpr int SH = 5 - Log2<SCAN_U * NQ>::v;
  const int vi = lane >> SH;           // value index u*NQ+q held by this lane
  const int my_q = vi % NQ;
  const int64_t my_r = r0 + vi / NQ;
  unsigned long long wq = worst[0];
#pragma unroll
  for (int q = 1; q < NQ; q++) if (my_q == q) wq = worst[q];
  const unsigned long long key = make_key(s, (uint32_t)my_r);
  const bool live = ((lane & ((1 << SH) - 1)) == 0) && my_r < n && my_q < nq_valid && (s == s);
  warp_offer<NQ, SH>(wkeys, k, live && key > wq, key, worst, worst_pos, lane);
}

template <int NQ, int CH>
__global__ void __launch_bounds__(256)
flat_scan_kernel(const uint4* __restrict__ X, int64_t n, int cpr, const float* __restrict__ Q, int nq_valid,
                 int k, unsigned long long* __restrict__ out_keys, int64_t out_stride_q) {
  extern __shared__ unsigned long long s_keys[];  // [warps][NQ][k]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  unsigned long long* wkeys = s_keys + (size_t)warp * NQ * k;
  warp_lists_clear(wkeys, NQ * k, lane);
  __syncwarp();

  float qr[NQ][CH][8];
  const int d = cpr * 8;
#pragma unroll
  for (int q = 0; q < NQ; q++) load_query_slice<CH>(qr[q], Q + (size_t)q * d, cpr, lane, q < nq_valid);

  unsigned long long worst[NQ];
  int worst_pos[NQ];
#pragma unroll
  for (int q = 0; q < NQ; q++) { worst[q] = 0ull; worst_pos[q] = 0; }

  constexpr int V = SCAN_U * NQ;
  const int64_t gw = (int64_t)blockIdx.x * nwarps + warp;
  const int64_t total = (int64_t)gridDim.x * nwarps;
  const int64_t nblk = (n + SCAN_U - 1) / SCAN_U;

  for (int64_t blk = gw; blk < nblk; blk += total) {
    const int64_t r0 = blk * SCAN_U;
    uint4 v[SCAN_U][CH];
#pragma unroll
    for (int u = 0; u < SCAN_U; u++) {
#pragma unroll
      for (int c = 0; c < CH; c++) {
        const int ci = c * 32 + lane;
        if (r0 + u < n && ci < cpr) v[u][c] = ld_nc_v4(X + (r0 + u) * cpr + ci);
        else v[u][c] = make_uint4(0u, 0u, 0u, 0u);
      }
    }
    float acc[V];
#pragma unroll
    for (int i = 0; i < V; i++) acc[i] = 0.0f;
#pragma unroll
    for (int u = 0; u < SCAN_U; u++) {
#pragma unroll
      for (int c = 0; c < CH; c++) {
        float f[8];
        chunk_to_f32(v[u][c], f);
#pragma unroll
        for (int q = 0; q < NQ; q++) fma_chunk(f, qr[q][c], acc[u * NQ + q]);
      }
    }
    warp_transpose_reduce<V>(acc, lane);
    offer_block_scores<NQ>(acc[0], r0, n, nq_valid, wkeys, k, worst, worst_pos, lane);
  }
  __syncwarp();
#pragma unroll
  for (int q = 0; q < NQ; q++)
    if (q < nq_valid) warp_list_store(out_keys + (int64_t)q * out_stride_q + gw * k, wkeys + q * k, k, lane);
}

// ---- staged variant: cp.async.bulk ring -------------------------------------------------------------
// Same arithmetic and the same per-warp candidate lists, but the rows reach the SM through a
// shared-memory ring filled by 1-D bulk async copies (one elected producer thread, one mbarrier
// per slot), so the bytes in flight per SM (STAGES x 32 rows x 2d bytes, ~190 KB) no longer depend
// on how many loads the register file can hold.  One CTA per SM: 8 consumer warps + 1 producer.
constexpr int TS_ROWS = 32;       // rows per slot (4 per consumer warp)
constexpr int TS_CONSUMERS = 8;   // consumer warps

__device__ __forceinline__ void bulk_copy_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   (uint32_t)__cvta_generic_to_shared(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"((uint32_t)__cvta_generic_to_shared(bar))
               : "memory");
}
__device__ __forceinline__ void ts_mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void ts_mbar_expect(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void ts_mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"((uint32_t)__cvta_generic_to_shared(bar)) : "memory");
}
__device__ __forceinline__ void ts_mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile(
        "{\n\t.reg .pred P;\n\tmbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\tselp.b32 %0, 1, 0, P;\n\t}\n"
        : "=r"(ok)
        : "r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(parity)
        : "memory");
  }
}

template <int NQ, int CH>
__global__ void __launch_bounds__((TS_CONSUMERS + 1) * 32, 1)
flat_scan_staged_kernel(const uint4* __restrict__ X, int64_t n, int cpr, const float* __restrict__ Q, int nq_valid,
                        int k, int stages, unsigned long long* __restrict__ out_keys, int64_t out_stride_q) {
  extern __shared__ __align__(128) unsigned char ts_smem[];
  const int row_bytes = cpr * 16;
  const int slot_bytes = TS_ROWS * row_bytes;
  unsigned char* ring = ts_smem;                                                          // [stages][slot_bytes]
  unsigned long long* s_keys = reinterpret_cast<unsigned long long*>(ts_smem + (size_t)stages * slot_bytes);  // [8][NQ][k]
  uint64_t* full = reinterpret_cast<uint64_t*>(s_keys + (size_t)TS_CONSUMERS * NQ * k);
  uint64_t* empty = full + stages;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; s++) {
      ts_mbar_init(&full[s], 1);
      ts_mbar_init(&empty[s], TS_CONSUMERS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int64_t nblocks = (n + TS_ROWS - 1) / TS_ROWS;

  if (warp == TS_CONSUMERS) {
    // ---------------- producer ----------------
    if (lane == 0) {
      int s = 0;
      uint32_t phase = 0;
      for (int64_t b = blockIdx.x; b < nblocks; b += gridDim.x) {
        ts_mbar_wait(&empty[s], phase ^ 1);
        const int64_t r0 = b * TS_ROWS;
        const int rows = (int)((n - r0) < TS_ROWS ? (n - r0) : TS_ROWS);
        const uint32_t bytes = (uint32_t)rows * (uint32_t)row_bytes;
        ts_mbar_expect(&full[s], bytes);
        bulk_copy_g2s(ring + (size_t)s * slot_bytes, X + r0 * cpr, bytes, &full[s]);
        if (++s == stages) { s = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ---------------- consumers ----------------
  unsigned long long* wkeys = s_keys + (size_t)warp * NQ * k;
  warp_lists_clear(wkeys, NQ * k, lane);
  __syncwarp();
  float qr[NQ][CH][8];
  const int d = cpr * 8;
#pragma unroll
  for (int q = 0; q < NQ; q++) load_query_slice<CH>(qr[q], Q + (size_t)q * d, cpr, lane, q < nq_valid);
  unsigned long long worst[NQ];
  int worst_pos[NQ];
#pragma unroll
  for (int q = 0; q < NQ; q++) { worst[q] = 0ull; worst_pos[q] = 0; }
  constexpr int V = SCAN_U * NQ;

  int s = 0;
  uint32_t phase = 0;
  for (int64_t b = blockIdx.x; b < nblocks; b += gridDim.x) {
    ts_mbar_wait(&full[s], phase);
    const uint4* slot = reinterpret_cast<const uint4*>(ring + (size_t)s * slot_bytes);
    const int64_t r0 = b * TS_ROWS + warp * SCAN_U;
    float acc[V];
#pragma unroll
    for (int i = 0; i < V; i++) acc[i] = 0.0f;
#pragma unroll
    for (int u = 0; u < SCAN_U; u++) {
#pragma unroll
      for (int c = 0; c < CH; c++) {
        const int ci = c * 32 + lane;
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if (r0 + u < n && ci < cpr) v = slot[(warp * SCAN_U + u) * cpr + ci];
        float f[8];
        chunk_to_f32(v, f);
#pragma unroll
        for (int q = 0; q < NQ; q++) fma_chunk(f, qr[q][c], acc[u * NQ + q]);
      }
    }
    // the slot's bytes are in registers: hand it back to the producer before the reduction
    __syncwarp();
    if (lane == 0) ts_mbar_arrive(&empty[s]);
    if (++s == stages) { s = 0; phase ^= 1; }

    warp_transpose_reduce<V>(acc, lane);
    offer_block_scores<NQ>(acc[0], r0, n, nq_valid, wkeys, k, worst, worst_pos, lane);
  }
  __syncwarp();
  const int64_t gw = (int64_t)blockIdx.x * TS_CONSUMERS + warp;
#pragma unroll
  for (int q = 0; q < NQ; q++)
    if (q < nq_valid) warp_list_store(out_keys + (int64_t)q * out_stride_q + gw * k, wkeys + q * k, k, lane);
}

// Select the k best of M candidate keys per query: grid (slices, nq); every block streams its
// slice through a C-entry shared buffer, keeping a sorted top-k at the front.
__global__ void __launch_bounds__(1024)
topk_select_kernel(const unsigned long long* __restrict__ in, int64_t in_stride_q, int64_t M, int k, int C,
                   unsigned long long* __restrict__ out, int64_t out_stride_q) {
  extern __shared__ unsigned long long buf[];
  const int q = blockIdx.y, s = blockIdx.x, slices = gridDim.x;
  const int64_t per = (M + slices - 1) / slices;
  const int64_t begin = (int64_t)s * per;
  const int64_t end = begin + per < M ? begin + per : M;
  const unsigned long long* src = in + (int64_t)q * in_stride_q;
  int have = 0;
  int64_t pos = begin;
  do {
    const int fill = C - have;
    for (int i = threadIdx.x; i < fill; i += blockDim.x) {
      const int64_t idx = pos + i;
      buf[have + i] = idx < end ? src[idx] : 0ull;
    }
    pos += fill;
    __syncthreads();
    block_bitonic_sort_desc(buf, C);
    have = k;
  } while (pos < end);
  unsigned long long* o = out + (int64_t)q * out_stride_q + (int64_t)s * k;
  for (int j = threadIdx.x; j < k; j += blockDim.x) o[j] = buf[j];
}

__global__ void decode_keys_kernel(const unsigned long long* __restrict__ keys, int64_t count, int64_t id_base,
                                   const uint32_t* __restrict__ slot_to_id, float* __restrict__ D,
                                   int64_t* __restrict__ I) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const unsigned long long key = keys[i];
  if (key == 0ull) {
    D[i] = -FLT_MAX;
    I[i] = -1;
  } else {
    D[i] = key_score(key);
    uint32_t id = key_id(key);
    if (slot_to_id) id = slot_to_id[id];
    I[i] = id_base + (int64_t)id;
  }
}

// ---- host side ----------------------------------------------------------------------------------

int index_ws(b200_index* idx, int slot, size_t bytes, void** out) {
  if (idx->ws_bytes[slot] < bytes) {
    if (idx->ws[slot]) B200_CUDA(cudaFree(idx->ws[slot]));
    idx->ws[slot] = nullptr;
    idx->ws_bytes[slot] = 0;
    size_t want = bytes + (bytes >> 2);
    B200_CUDA(cudaMalloc(&idx->ws[slot], want));
    idx->ws_bytes[slot] = want;
  }
  *out = idx->ws[slot];
  return B200_OK;
}

int launch_topk_select(const unsigned long long* in, int64_t in_stride_q, int64_t M, int k, int C,
                       unsigned long long* out, int64_t out_stride_q, int slices, int nq, cudaStream_t st) {
  const size_t sel_smem = (size_t)C * 8;
  if (sel_smem > 48 * 1024)
    B200_CUDA(cudaFuncSetAttribute(topk_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sel_smem));
  topk_select_kernel<<<dim3(slices, nq), 1024, sel_smem, st>>>(in, in_stride_q, M, k, C, out, out_stride_q);
  B200_LAUNCH_OK();
  return B200_OK;
}

int plan_select(int64_t M, int k, SelectPlan* p) {
  p->M = M;
  p->k = k;
  p->C = select_buffer(k);
  B200_CHECK((size_t)p->C * 8 <= SELECT_SMEM_MAX, B200_ERR_UNSUPPORTED, "search: k=%d exceeds the supported maximum (8192)", k);
  // level 1: one sort round per block (a block sorts one C-entry chunk of the candidates) — the select of a single
  // query is latency, not throughput: dependent sort rounds per block are what it costs
  p->slices = (int)std::min<int64_t>(256, std::max<int64_t>(1, (M + p->C - 1) / p->C));
  p->C2 = std::min(p->C, std::max(next_pow2(2 * k), next_pow2(p->slices * k)));   // level 2 buffer: slices * k keys
  return B200_OK;
}

int select_topk(const SelectPlan& p, const unsigned long long* cand, unsigned long long* tmp, unsigned long long* out,
                int nq, cudaStream_t st) {
  const int64_t M2 = (int64_t)p.slices * p.k;
  // level 1: slices per query; level 2: one block per query
  B200_TRY(launch_topk_select(cand, p.M, p.M, p.k, p.C, tmp, M2, p.slices, nq, st));
  return launch_topk_select(tmp, M2, M2, p.k, p.C2, out, p.k, 1, nq, st);
}

typedef void (*scan_fn)(const uint4*, int64_t, int, const float*, int, int, unsigned long long*, int64_t);

template <int NQ>
static scan_fn pick_ch(int ch) {
  switch (ch) {
    case 1: return flat_scan_kernel<NQ, 1>;
    case 2: return flat_scan_kernel<NQ, 2>;
    case 3: return flat_scan_kernel<NQ, 3>;
  }
  if constexpr (NQ <= 2) {
    switch (ch) {
      case 4: return flat_scan_kernel<NQ, 4>;
      case 5: return flat_scan_kernel<NQ, 5>;
      case 6: return flat_scan_kernel<NQ, 6>;
    }
  }
  if constexpr (NQ == 1) {
    switch (ch) {
      case 7: return flat_scan_kernel<NQ, 7>;
      case 8: return flat_scan_kernel<NQ, 8>;
    }
  }
  return nullptr;
}
static scan_fn pick_scan(int nqp, int ch) {
  if (nqp == 4) return pick_ch<4>(ch);
  if (nqp == 2) return pick_ch<2>(ch);
  return pick_ch<1>(ch);
}

typedef void (*staged_fn)(const uint4*, int64_t, int, const float*, int, int, int, unsigned long long*, int64_t);
template <int NQ>
static staged_fn pick_staged_ch(int ch) {
  switch (ch) {
    case 1: return flat_scan_staged_kernel<NQ, 1>;
    case 2: return flat_scan_staged_kernel<NQ, 2>;
    case 3: return flat_scan_staged_kernel<NQ, 3>;
  }
  if constexpr (NQ <= 2) {
    if (ch == 4) return flat_scan_staged_kernel<NQ, 4>;
  }
  return nullptr;
}
static staged_fn pick_staged(int nqp, int ch) {
  if (nqp == 4) return pick_staged_ch<4>(ch);
  if (nqp == 2) return pick_staged_ch<2>(ch);
  return pick_staged_ch<1>(ch);
}

struct ScanPlan {
  int nqp;       // queries per pass
  int threads;   // block size
  int grid;
  size_t smem;
  scan_fn fn;
  staged_fn sfn = nullptr;  // cp.async.bulk ring variant (preferred when it fits)
  int stages = 0;
  int warps_out = 0;        // candidate lists written per block
};

static int plan_scan(const b200_index* idx, int k, int nq, ScanPlan* p) {
  const int ch = (idx->d / 8 + 31) / 32;
  // queries per pass: the FMA path stays HBM-bound up to ~2 queries per pass; 4 trades some
  // bandwidth for fewer passes when there are many queries.  nqp*ch bounds the query registers.
  int nqp = nq >= 4 ? 4 : (nq >= 2 ? 2 : 1);
  while (nqp > 1 && nqp * ch > 12) nqp >>= 1;
  int threads = 256;
  const size_t budget = 96 * 1024;  // keeps two blocks per SM
  while (nqp > 1 && (size_t)(threads / 32) * nqp * k * 8 > budget) nqp >>= 1;
  while (threads > 64 && (size_t)(threads / 32) * nqp * k * 8 > 200 * 1024) threads >>= 1;
  if ((size_t)(threads / 32) * nqp * k * 8 > 200 * 1024) {
    set_error("search: k=%d exceeds the supported maximum (8192)", k);
    return B200_ERR_UNSUPPORTED;
  }
  p->smem = (size_t)(threads / 32) * nqp * k * 8;
  p->fn = pick_scan(nqp, ch);
  if (!p->fn) {
    set_error("search: unsupported dimension d=%d", idx->d);
    return B200_ERR_UNSUPPORTED;
  }
  if (p->smem > 48 * 1024)
    B200_CUDA(cudaFuncSetAttribute((const void*)p->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem));
  int per_sm = 0;
  B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, (const void*)p->fn, threads, p->smem));
  if (per_sm < 1) per_sm = 1;
  if (per_sm > 4) per_sm = 4;
  p->nqp = nqp;
  p->threads = threads;
  p->grid = idx->sms * per_sm;
  p->warps_out = threads / 32;
  // staged variant: one block per SM, ring of 32-row slots in shared memory
  if (idx->use_staged) {
    const size_t slot = (size_t)TS_ROWS * idx->d * 2;
    const size_t lists = (size_t)TS_CONSUMERS * nqp * k * 8;
    const size_t fixed = lists + 256;
    const size_t budget = 220 * 1024;
    staged_fn sf = pick_staged(nqp, ch);
    if (sf && fixed + 3 * slot <= budget) {
      int stages = (int)std::min<size_t>(8, (budget - fixed) / slot);
      p->sfn = sf;
      p->stages = stages;
      p->smem = (size_t)stages * slot + fixed;
      p->threads = (TS_CONSUMERS + 1) * 32;
      p->grid = idx->sms;
      p->warps_out = TS_CONSUMERS;
      B200_CUDA(cudaFuncSetAttribute((const void*)sf, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem));
    }
  }
  return B200_OK;
}

int scan_topk_keys(b200_index* idx, const __half* rows, int64_t n, const float* d_q, int nq, int k,
                   unsigned long long* d_keys_out, cudaStream_t st) {
  const int d = idx->d;
  // many queries at once: one tensor-core pass per 128 queries instead of one FMA pass per 4
  if (idx->use_mma && nq > 4 && k <= 128 && n >= 4096 && n < (1ll << 31) && d >= 64)
    return scan_topk_keys_mma(idx, rows, n, d_q, nq, k, d_keys_out, st);
  ScanPlan p;
  B200_TRY(plan_scan(idx, k, nq, &p));
  idx->last_scan_plan[0] = p.sfn ? 1 : 0;
  idx->last_scan_plan[1] = p.nqp;
  idx->last_scan_plan[2] = (d / 8 + 31) / 32;
  idx->last_scan_plan[3] = p.stages;
  const int64_t total_warps = (int64_t)p.grid * p.warps_out;
  const int64_t M1 = total_warps * k;
  SelectPlan sel;
  B200_TRY(plan_select(M1, k, &sel));
  const int QB = 64;  // queries per batch (bounds the scratch)
  void* ws = nullptr;
  B200_TRY(index_ws(idx, 0, sel.keys(QB) * 8, &ws));
  unsigned long long* k1 = (unsigned long long*)ws;
  unsigned long long* k2 = k1 + (size_t)QB * M1;

  for (int q0 = 0; q0 < nq; q0 += QB) {
    const int qb = std::min(QB, nq - q0);
    B200_TRY(scan_timer_begin(idx, st));   // time the row-scan kernels of this batch
    for (int qq = 0; qq < qb; qq += p.nqp) {
      const int valid = std::min(p.nqp, qb - qq);
      const float* qptr = d_q + (size_t)(q0 + qq) * d;
      unsigned long long* kp = k1 + (size_t)qq * M1;
      if (p.sfn)
        p.sfn<<<p.grid, p.threads, p.smem, st>>>(reinterpret_cast<const uint4*>(rows), n, d / 8, qptr, valid, k, p.stages, kp, M1);
      else
        p.fn<<<p.grid, p.threads, p.smem, st>>>(reinterpret_cast<const uint4*>(rows), n, d / 8, qptr, valid, k, kp, M1);
      B200_LAUNCH_OK();
      idx->last_scan_launches++;
    }
    B200_TRY(scan_timer_end(idx, st));
    B200_TRY(select_topk(sel, k1, k2, d_keys_out + (size_t)q0 * k, qb, st));
  }
  return B200_OK;
}

int decode_keys(const unsigned long long* keys, int64_t count, int64_t id_base, const uint32_t* slot_to_id, float* D,
                int64_t* I, cudaStream_t st) {
  if (count == 0) return B200_OK;
  decode_keys_kernel<<<(unsigned)((count + 255) / 256), 256, 0, st>>>(keys, count, id_base, slot_to_id, D, I);
  B200_LAUNCH_OK();
  return B200_OK;
}

}  // namespace b200

// ---- range search (index.range_search: clip_filter.py:52, clip_back.py:294) ---------------------------
// All rows whose score with the query exceeds `thresh`: same warp-per-4-rows scan, hits appended
// to a global (row, score) list per query through one atomic counter.  Results are unordered (FAISS
// leaves the order within a query unspecified); the host wrapper sorts them by id.
namespace b200 {

template <int CH>
__global__ void __launch_bounds__(256)
range_scan_kernel(const uint4* __restrict__ X, int64_t n, int cpr, const float* __restrict__ Q, float thresh,
                  unsigned long long* __restrict__ out, unsigned int cap, unsigned int* __restrict__ counter) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  float qr[CH][8];
  load_query_slice<CH>(qr, Q, cpr, lane, true);
  const int64_t gw = (int64_t)blockIdx.x * nwarps + warp, total = (int64_t)gridDim.x * nwarps;
  const int64_t nblk = (n + 3) / 4;
  for (int64_t blk = gw; blk < nblk; blk += total) {
    const int64_t r0 = blk * 4;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int u = 0; u < 4; u++) {
#pragma unroll
      for (int c = 0; c < CH; c++) {
        const int ci = c * 32 + lane;
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if (r0 + u < n && ci < cpr) v = ld_nc_v4(X + (r0 + u) * cpr + ci);
        fma_chunk(v, qr[c], acc[u]);
      }
    }
    warp_transpose_reduce<4>(acc, lane);
    const int64_t my_r = r0 + (lane >> 3);
    if ((lane & 7) == 0 && my_r < n && acc[0] > thresh) range_append(out, cap, counter, acc[0], (uint32_t)my_r);
  }
}

typedef void (*range_fn)(const uint4*, int64_t, int, const float*, float, unsigned long long*, unsigned int, unsigned int*);
static range_fn pick_range(int ch) {
  switch (ch) {
    case 1: return range_scan_kernel<1>;
    case 2: return range_scan_kernel<2>;
    case 3: return range_scan_kernel<3>;
    case 4: return range_scan_kernel<4>;
    case 5: return range_scan_kernel<5>;
    case 6: return range_scan_kernel<6>;
    case 7: return range_scan_kernel<7>;
    case 8: return range_scan_kernel<8>;
  }
  return nullptr;
}

// One query: appends up to `cap` keys to d_out, *d_count receives the number of hits (may exceed cap).
int range_scan(b200_index* idx, const __half* rows, int64_t n, const float* d_q, float thresh, unsigned long long* d_out,
               unsigned int cap, unsigned int* d_count, cudaStream_t st) {
  const int ch = (idx->d / 8 + 31) / 32;
  range_fn fn = pick_range(ch);
  B200_CHECK(fn != nullptr, B200_ERR_UNSUPPORTED, "range_search: unsupported dimension %d", idx->d);
  B200_CUDA(cudaMemsetAsync(d_count, 0, sizeof(unsigned int), st));
  fn<<<idx->sms * 4, 256, 0, st>>>(reinterpret_cast<const uint4*>(rows), n, idx->d / 8, d_q, thresh, d_out, cap, d_count);
  B200_LAUNCH_OK();
  return B200_OK;
}

}  // namespace b200
