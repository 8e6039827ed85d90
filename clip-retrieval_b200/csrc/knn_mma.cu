// Search path, batched exhaustive scan on the tensor cores: the same answer as flat_scan_kernel
// (knn_scan.cu) when many queries arrive together (BASELINE configs[2]: 1000 queries, top-40), with
// the index read once per 128 queries instead of once per 4.
//
//   S[row, q] = sum_j X[row, j] * Q[q, j]          X fp16 rows (HBM), Q fp32 queries
//
// wgmma with fp16 operands needs the query in fp16, and rounding it (2^-11 relative) would swap
// near-tied neighbours, so each fp32 query is split into two fp16 rows: hi = fp16(q) and
// lo = fp16((q - hi) * 2^11); the products with fp16 rows are exact in fp32, the two partial sums
// are accumulated in separate accumulator columns and recombined as s = s_hi + s_lo * 2^-11 in the
// epilogue (22 significant bits of the query: below the fp32 accumulation noise already accepted
// for the FMA kernel).
//
// Structure = the GEMM core (gemm.cuh): warp 4 TMA producer (X box 64x64, Q' box 256x64, 128B
// swizzle, 5-stage ring), warps 0..3 one consumer warpgroup issuing wgmma m64n256k16 over the 64
// rows of the tile with the accumulator in registers (128 fp32 per thread: with five warps per CTA no
// SM sub-partition holds more than two of them, which leaves room for it).  A CTA owns whole 64-row tiles
// (tile = cta + i*ctas) and walks all query groups of a tile back to back, so the X tile is re-read
// from L2, not HBM.  Epilogue, in the accumulator's own register layout: a score that reaches the
// query's current threshold is appended to the (CTA, query) candidate buffer (atomic counter in
// shared memory, buffer in global/L2); buffers are compacted to their k best by the consumer warps
// between groups, which raises the threshold.  A final select merges the CTAs.
// Thresholds are warmed up by two sampling passes (one row tile per CTA, then every 32nd row
// tile: the k-th best score of a subset is a valid lower bound for the full set), so the full pass
// almost never takes the append path.
// Roofline: tensor pipe (4*N*d*nq flops with the split) for large nq, HBM (N*d*2 bytes per 128
// queries) below ~64 queries per pass; every further 128-query group costs the same tensor time again.
//
// Above 128 queries the split is therefore the cost, and the kernel has a second mode (HILO =
// false): only the hi halves are multiplied (256 queries per group, half the flops), which yields
// APPROXIMATE scores with a known bound |s - s_hi| <= ||q - fp16(q)||_2 * max_row ||x||_2.  That pass
// keeps 2k candidates per query; they are re-scored exactly (fp32 FMA over the fp16 row), the best k
// are kept, and the result is PROVEN exact per query by checking that the worst kept candidate of the
// approximate pass, plus the bound, is still below the k-th exact score — any row that was not a
// candidate is then strictly worse than the k-th result.  Queries that fail the proof (near-duplicate
// rows packed inside the bound) are re-run through the split mode.  Ids therefore stay exact.
#include "index.cuh"
#include "topk.cuh"
#include "ptx.cuh"
#include "gemm.cuh"
#include <algorithm>
#include <stdlib.h>

namespace b200 {

int launch_topk_select(const unsigned long long* in, int64_t in_stride_q, int64_t M, int k, int C,
                       unsigned long long* out, int64_t out_stride_q, int slices, int nq, cudaStream_t st);

constexpr int MS_BM = 64;        // rows per tile
constexpr int MS_QG = 128;       // queries per group (256 MMA columns: hi | lo)
constexpr int MS_BN = 256;
constexpr int MS_BK = 64;
constexpr int MS_STAGES = 5;
constexpr int MS_CAP = 512;      // candidate buffer entries per (CTA, query)
constexpr int MS_KMAX = 128;     // k supported by this path
constexpr int MS_THREADS = 160;   // warps 0..3: the consumer warpgroup, warp 4: TMA producer
constexpr int MS_WARP_TMA = 4;
constexpr int MS_CONSUMERS = 128;
constexpr int MS_A_BYTES = MS_BM * MS_BK * 2;
constexpr int MS_B_BYTES = MS_BN * MS_BK * 2;
constexpr int MS_STAGE_BYTES = MS_A_BYTES + MS_B_BYTES;

// fp32 queries -> fp16 [groups*256, d].  Split mode: row g*256 + c (c < 128) = hi of query
// g*128 + c, row g*256 + 128 + c = lo * 2^11 of the same query.  Hi-only mode: row q = fp16(query q).
// Padding queries are zero rows.
template <bool HILO>
__global__ void split_queries_kernel(const float* __restrict__ Q, int nq, int d, __half* __restrict__ Qp, int groups) {
  constexpr int QG = HILO ? MS_QG : MS_BN;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t total = (int64_t)groups * QG * d;
  if (i >= total) return;
  const int q = (int)(i / d), j = (int)(i - (int64_t)q * d);
  float v = q < nq ? Q[(int64_t)q * d + j] : 0.0f;
  const __half hi = __float2half_rn(v);
  if constexpr (HILO) {
    const int g = q / MS_QG, c = q - g * MS_QG;
    const __half lo = __float2half_rn((v - __half2float(hi)) * 2048.0f);
    Qp[((int64_t)g * MS_BN + c) * d + j] = hi;
    Qp[((int64_t)g * MS_BN + MS_QG + c) * d + j] = lo;
  } else {
    Qp[(int64_t)q * d + j] = hi;
  }
}

// ---- hi-only mode: error bound, exact re-scoring, proof, fallback list ----------------------------
// One warp per query: margin[q] = ||q - fp16(q)||_2 * R + 1e-5 * ||q||_2 * R, R = max row norm.  The
// second term covers the fp32 accumulation noise of the two score computations being compared.
__global__ void query_margin_kernel(const float* __restrict__ Q, int nq, int d, const float* __restrict__ row_norm2_max,
                                    float* __restrict__ margin) {
  const int q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (q >= nq) return;
  float r2 = 0.f, n2 = 0.f;
  for (int j = lane; j < d; j += 32) {
    const float v = Q[(int64_t)q * d + j];
    const float e = v - __half2float(__float2half_rn(v));
    r2 = fmaf(e, e, r2);
    n2 = fmaf(v, v, n2);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    r2 += __shfl_xor_sync(FULL, r2, o);
    n2 += __shfl_xor_sync(FULL, n2, o);
  }
  if (lane == 0) {
    const float R = sqrtf(*row_norm2_max) * 1.0001f;
    margin[q] = (sqrtf(r2) * 1.0001f + 1e-5f * sqrtf(n2)) * R;
  }
}

// max over rows of ||x||^2 (fp32), one warp per row, grid-stride; result through atomicMax on the
// bit pattern (non-negative floats order like unsigned integers).  NaN/Inf rows yield +Inf -> the
// margin becomes infinite and every query takes the split mode.
__global__ void row_norm2_max_kernel(const uint4* __restrict__ X, int64_t n, int cpr, unsigned int* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t gw = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, total = ((int64_t)gridDim.x * blockDim.x) >> 5;
  float best = 0.f;
  for (int64_t r = gw; r < n; r += total) {
    float a = 0.f;
    for (int c = lane; c < cpr; c += 32) {
      const uint4 v = ld_nc_v4(X + r * cpr + c);
      const __half2* h2 = reinterpret_cast<const __half2*>(&v);
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const float2 t = __half22float2(h2[j]);
        a = fmaf(t.x, t.x, a);
        a = fmaf(t.y, t.y, a);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(FULL, a, o);
    if (!(a <= 3.0e38f)) a = INFINITY;   // NaN or overflow
    best = fmaxf(best, a);
  }
  if (lane == 0) atomicMax(out, __float_as_uint(best));
}

// One warp per (query, candidate): exact fp32 score of the candidate row, re-keyed.
__global__ void rescore_kernel(const uint4* __restrict__ X, int cpr, const float* __restrict__ Q, int d,
                               const unsigned long long* __restrict__ approx, int64_t count, int kc,
                               unsigned long long* __restrict__ exact) {
  const int lane = threadIdx.x & 31;
  const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (w >= count) return;
  const unsigned long long key = approx[w];
  if (key == 0ull) {
    if (lane == 0) exact[w] = 0ull;
    return;
  }
  const uint32_t id = key_id(key);
  const float* q = Q + (w / kc) * d;
  float a = 0.f;
  for (int c = lane; c < cpr; c += 32) {
    const uint4 v = ld_nc_v4(X + (int64_t)id * cpr + c);
    const float4 q0 = *reinterpret_cast<const float4*>(q + c * 8);
    const float4 q1 = *reinterpret_cast<const float4*>(q + c * 8 + 4);
    const __half2* h2 = reinterpret_cast<const __half2*>(&v);
    const float2 t0 = __half22float2(h2[0]), t1 = __half22float2(h2[1]), t2 = __half22float2(h2[2]),
                 t3 = __half22float2(h2[3]);
    a = fmaf(t0.x, q0.x, a); a = fmaf(t0.y, q0.y, a); a = fmaf(t1.x, q0.z, a); a = fmaf(t1.y, q0.w, a);
    a = fmaf(t2.x, q1.x, a); a = fmaf(t2.y, q1.y, a); a = fmaf(t3.x, q1.z, a); a = fmaf(t3.y, q1.w, a);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(FULL, a, o);
  if (lane == 0) exact[w] = (a == a) ? make_key(a, id) : 0ull;
}

// Proof per query; failing queries are appended to fail_list (fail_count = its length).
__global__ void verify_kernel(const unsigned long long* __restrict__ approx, int kc,
                              const unsigned long long* __restrict__ result, int k, const float* __restrict__ margin,
                              int nq, int* __restrict__ fail_list, int* __restrict__ fail_count) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nq) return;
  const unsigned long long worst_kept = approx[(int64_t)q * kc + (kc - 1)];
  const unsigned long long kth = result[(int64_t)q * k + (k - 1)];
  bool ok;
  if (worst_kept == 0ull) ok = true;           // fewer than kc scorable rows exist: all of them were candidates
  else if (kth == 0ull) ok = false;
  else ok = key_score(worst_kept) + margin[q] < key_score(kth);
  if (!ok) fail_list[atomicAdd(fail_count, 1)] = q;
}

__global__ void gather_queries_kernel(const float* __restrict__ Q, int d, const int* __restrict__ list, int count,
                                      float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)count * d) return;
  const int r = (int)(i / d), j = (int)(i - (int64_t)r * d);
  out[i] = Q[(int64_t)list[r] * d + j];
}
__global__ void scatter_keys_kernel(const unsigned long long* __restrict__ in, int k, const int* __restrict__ list,
                                    int count, unsigned long long* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)count * k) return;
  const int r = (int)(i / k), j = (int)(i - (int64_t)r * k);
  out[(int64_t)list[r] * k + j] = in[i];
}

// thr[q] = score of the k-th selected key of a sampling pass (a lower bound on the final k-th best)
__global__ void kth_score_kernel(const unsigned long long* __restrict__ keys, int nq, int k, float* __restrict__ thr) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nq) return;
  const unsigned long long kk = keys[(int64_t)q * k + (k - 1)];
  thr[q] = kk != 0ull ? key_score(kk) : -INFINITY;
}

// Keep the k best of a (CTA, query) candidate buffer (unsorted, in place, buf[0..k)); returns the
// new threshold score.  One warp, the keys live in registers (MS_CAP/32 per lane).  The k-th largest
// key is found by a most-significant-bit-first radix select (one warp-wide popcount per bit), then
// the survivors are packed with ballot prefix sums — no sorting, ~2.5k cycles instead of ~20k.
__device__ __forceinline__ float compact_buffer(unsigned long long* buf, int count, int k, int lane) {
  constexpr int R = MS_CAP / 32;
  unsigned long long v[R];
#pragma unroll
  for (int i = 0; i < R; i++) {
    const int j = i * 32 + lane;
    v[i] = j < count ? buf[j] : 0ull;
  }
  __syncwarp();
  if (count <= k) return -INFINITY;
  // radix select: `prefix` = the bits of the k-th largest key decided so far
  unsigned long long prefix = 0ull, decided = 0ull;
  int need = k;  // rank still to locate among keys matching the prefix
  for (int bit = 63; bit >= 0; bit--) {
    const unsigned long long b = 1ull << bit;
    int c = 0;
#pragma unroll
    for (int i = 0; i < R; i++) c += ((v[i] & decided) == prefix && (v[i] & b)) ? 1 : 0;
    c = __reduce_add_sync(FULL, c);
    if (c >= need) prefix |= b;   // the k-th largest has this bit set
    else need -= c;               // skip the c keys above, continue among those with the bit clear
    decided |= b;
  }
  const unsigned long long kth = prefix;  // keys are unique, so exactly k keys are >= kth
  int base = 0;
#pragma unroll
  for (int i = 0; i < R; i++) {
    const bool keep = v[i] >= kth && v[i] != 0ull;
    const unsigned m = __ballot_sync(FULL, keep);
    if (keep) buf[base + __popc(m & ((1u << lane) - 1u))] = v[i];
    base += __popc(m);
  }
  __syncwarp();
  return kth != 0ull ? key_score(kth) : -INFINITY;
}

template <bool HILO>
__global__ void __launch_bounds__(MS_THREADS, 1)
scan_mma_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmQ, int64_t n, int d,
                int nq, int groups, int k, unsigned long long* __restrict__ cand /* [grid][groups*128][CAP] */,
                unsigned long long* __restrict__ dense /* [nq][grid][k] */, int tile_stride,
                const float* __restrict__ thr_init /* [nq] lower bounds on the k-th best score, or null */) {
  constexpr int QG = HILO ? MS_QG : MS_BN;   // queries per group: 128 (hi | lo columns) or 256 (hi only)
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = ptx::smem_u32(smem_raw);
  uint8_t* base = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* sA = base;
  uint8_t* sB = base + MS_STAGES * MS_A_BYTES;
  float* s_thr = reinterpret_cast<float*>(base + MS_STAGES * MS_STAGE_BYTES);  // [groups*QG]
  int* s_cnt = reinterpret_cast<int*>(s_thr + groups * QG);                    // [groups*QG]
  uint64_t* full = reinterpret_cast<uint64_t*>(s_cnt + groups * QG);
  uint64_t* empty = full + MS_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t row_tiles = (n + MS_BM - 1) / MS_BM;
  const int kb = (d + MS_BK - 1) / MS_BK;

  for (int i = threadIdx.x; i < groups * QG; i += blockDim.x) {
    s_thr[i] = (thr_init != nullptr && i < nq) ? thr_init[i] : -INFINITY;
    s_cnt[i] = 0;
  }
  if (threadIdx.x == 0) {
    for (int st = 0; st < MS_STAGES; st++) {
      ptx::mbar_init(&full[st], 1);
      ptx::mbar_init(&empty[st], 4);   // one arrive per consumer warp
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (warp == MS_WARP_TMA) {
    if (lane == 0) {
      ptx::prefetch_tensormap(&tmX);
      ptx::prefetch_tensormap(&tmQ);
      int stage = 0;
      uint32_t phase = 0;
      for (int64_t rt = (int64_t)blockIdx.x * tile_stride; rt < row_tiles; rt += (int64_t)gridDim.x * tile_stride) {
        for (int g = 0; g < groups; g++) {
          for (int kbi = 0; kbi < kb; kbi++) {
            ptx::mbar_wait(&empty[stage], phase ^ 1);
            ptx::mbar_arrive_expect_tx(&full[stage], MS_STAGE_BYTES);
            ptx::tma_load_2d(sA + stage * MS_A_BYTES, &tmX, &full[stage], kbi * MS_BK, (int32_t)(rt * MS_BM));
            ptx::tma_load_2d(sB + stage * MS_B_BYTES, &tmQ, &full[stage], kbi * MS_BK, g * MS_BN);
            if (++stage == MS_STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  // ---------------- consumers: wgmma, thresholded append, compaction ----------------
  int stage = 0;
  uint32_t phase = 0;
  unsigned long long* my_cand = cand + (int64_t)blockIdx.x * groups * QG * MS_CAP;
  float acc[MS_BN / 2];
  for (int64_t rt = (int64_t)blockIdx.x * tile_stride; rt < row_tiles; rt += (int64_t)gridDim.x * tile_stride) {
    // accumulator rows of this thread: r0 and r0 + 8
    const int64_t r0 = rt * MS_BM + warp * 16 + (lane >> 2);
    for (int g = 0; g < groups; g++) {
      int prev = -1;
      for (int kbi = 0; kbi < kb; kbi++) {
        ptx::mbar_wait(&full[stage], phase);
        ptx::wgmma_fence();
        const uint64_t da = ptx::wgmma_desc_k_sw128(ptx::smem_u32(sA + stage * MS_A_BYTES));
        const uint64_t db = ptx::wgmma_desc_k_sw128(ptx::smem_u32(sB + stage * MS_B_BYTES));
#pragma unroll
        for (int kk = 0; kk < MS_BK / 16; kk++)
          ptx::wgmma_m64n256k16_f16(acc, da + (uint64_t)(kk * 2), db + (uint64_t)(kk * 2), (kbi | kk) != 0 ? 1u : 0u);
        ptx::wgmma_commit();
        // the group of the previous k-block has completed: its ring slot may be refilled
        ptx::wgmma_wait<1>();
        if (prev >= 0 && lane == 0) ptx::mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == MS_STAGES) { stage = 0; phase ^= 1; }
      }
      ptx::wgmma_wait<0>();
      ptx::fence_regs(acc);
      if (lane == 0) ptx::mbar_arrive(&empty[prev]);

      // register i of this thread: row r0 + 8 * ((i / 2) % 2), column 8 * (i / 4) + 2 * (lane % 4) + i % 2; in split
      // mode column c < 128 holds the hi product of query c and column c + 128 its lo product.
#pragma unroll
      for (int j = 0; j < QG / 8; j++) {
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const int col = 8 * j + 2 * (lane & 3) + e;
          const int q = g * QG + col;
          if (q >= nq) continue;
          const float th = s_thr[q];
#pragma unroll
          for (int h = 0; h < 2; h++) {
            float sc = acc[4 * j + 2 * h + e];
            if constexpr (HILO) sc = fmaf(acc[4 * (j + MS_QG / 8) + 2 * h + e], 1.0f / 2048.0f, sc);
            const int64_t row = r0 + 8 * h;
            if (sc >= th && row < n) {
              const int pos = atomicAdd(&s_cnt[q], 1);
              if (pos < MS_CAP) my_cand[(int64_t)q * MS_CAP + pos] = make_key(sc, (uint32_t)row);
            }
          }
        }
      }
      // compaction of this group's buffers that could overflow during the next tile
      const int gq = min(QG, nq - g * QG);   // live queries of this group
      __threadfence_block();
      asm volatile("bar.sync 1, %0;" ::"n"(MS_CONSUMERS) : "memory");
      // each warp owns 32 queries of the group; one lane-parallel look at their counters (the common case
      // — nothing close to overflowing — costs one shared load and a ballot instead of 32 dependent loads)
      for (int qb = warp * 32; qb < gq; qb += MS_CONSUMERS) {
        const int ql = qb + lane;
        const int my_cnt = ql < gq ? s_cnt[g * QG + ql] : 0;
        unsigned need = __ballot_sync(FULL, my_cnt > MS_CAP - MS_BM);
        while (need) {
          const int b = __ffs(need) - 1;
          need &= need - 1;
          const int q = g * QG + qb + b;
          const int cnt = __shfl_sync(FULL, my_cnt, b);
          const float thr = compact_buffer(my_cand + (int64_t)q * MS_CAP, min(cnt, MS_CAP), k, lane);
          if (lane == 0) {
            s_cnt[q] = min(cnt, k);
            if (thr > s_thr[q]) s_thr[q] = thr;
          }
        }
      }
      asm volatile("bar.sync 1, %0;" ::"n"(MS_CONSUMERS) : "memory");
    }
  }
  // final pass: every (CTA, query) buffer reduced to its k best and written densely for the merge
  for (int q = warp; q < nq; q += MS_CONSUMERS / 32) {
    unsigned long long* buf = my_cand + (int64_t)q * MS_CAP;
    const int cnt = s_cnt[q];
    if (cnt > k) compact_buffer(buf, min(cnt, MS_CAP), k, lane);
    const int have = min(cnt, k);   // slots past `have` were never written: emit the empty key
    unsigned long long* o = dense + ((int64_t)q * gridDim.x + blockIdx.x) * k;
    for (int j = lane; j < k; j += 32) o[j] = j < have ? buf[j] : 0ull;
  }
}

int make_tmap_2d(CUtensorMap* out, const void* ptr, int dtype_bf16, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                 uint32_t box_rows, uint32_t box_cols);

// One mode of the batched scan: k sorted keys per query into d_keys_out.
template <bool HILO>
static int scan_mma_passes(b200_index* idx, const __half* rows, int64_t n, const float* d_q, int nq, int k,
                           unsigned long long* d_keys_out, cudaStream_t st) {
  constexpr int QG = HILO ? MS_QG : MS_BN;
  const int d = idx->d;
  const int grid = idx->sms;
  const int QMAX = 1024;  // queries per launch (thresholds/counters live in shared memory)
  for (int q0 = 0; q0 < nq; q0 += QMAX) {
    const int nqb = std::min(QMAX, nq - q0);
    const int groups = (nqb + QG - 1) / QG;
    const size_t qp_bytes = ((size_t)groups * MS_BN * d * sizeof(__half) + 255) & ~(size_t)255;
    const size_t cand_bytes = (size_t)grid * groups * QG * MS_CAP * 8;
    const size_t dense_bytes = (size_t)nqb * grid * k * 8;
    void* ws = nullptr;
    B200_TRY(index_ws(idx, 0, qp_bytes + cand_bytes + dense_bytes + (size_t)nqb * 4 + 256, &ws));
    __half* Qp = (__half*)ws;
    unsigned long long* cand = (unsigned long long*)((char*)ws + qp_bytes);
    unsigned long long* dense = (unsigned long long*)((char*)ws + qp_bytes + cand_bytes);
    float* thr = (float*)((char*)ws + qp_bytes + cand_bytes + dense_bytes);   // (slot 3 belongs to the IVF caller)
    {
      const int64_t total = (int64_t)groups * QG * d;
      split_queries_kernel<HILO><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(d_q + (size_t)q0 * d, nqb, d, Qp, groups);
      B200_LAUNCH_OK();
    }
    CUtensorMap tmX, tmQ;
    B200_TRY(make_tmap_2d(&tmX, rows, 0, (uint64_t)n, (uint64_t)d, (uint64_t)d, MS_BM, MS_BK));
    B200_TRY(make_tmap_2d(&tmQ, Qp, 0, (uint64_t)groups * MS_BN, (uint64_t)d, (uint64_t)d, MS_BN, MS_BK));
    const size_t smem = (size_t)MS_STAGES * MS_STAGE_BYTES + (size_t)groups * QG * 8 + 256 + 1024;
    B200_CUDA(cudaFuncSetAttribute(scan_mma_kernel<HILO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if ((int)idx->ev.size() < idx->ev_used + 2) {
      cudaEvent_t a, b;
      B200_CUDA(cudaEventCreate(&a));
      B200_CUDA(cudaEventCreate(&b));
      idx->ev.push_back(a);
      idx->ev.push_back(b);
    }
    // sampling passes first (strided row tiles), each seeding the next pass's thresholds
    const int64_t row_tiles = (n + MS_BM - 1) / MS_BM;
    const int64_t M = (int64_t)grid * k;
    int C = 2048;
    while (C < 2 * k) C <<= 1;
    unsigned long long* keys_q = d_keys_out + (size_t)q0 * k;
    // Pass schedule.  The first pass starts from -inf thresholds, where EVERY score is appended and the
    // buffers are compacted every third tile, so it is kept to one tile per CTA (a sample of ctas*64 rows, no
    // compaction before the final one); its k-th best scores seed a 1/32 pass, whose k-th best scores seed the
    // full pass.
    const int64_t ctas = grid;
    int strides[3], npass = 0;
    if (row_tiles >= 8 * ctas) strides[npass++] = (int)std::min<int64_t>(row_tiles / ctas, 1 << 30);
    if (npass == 1 && strides[0] > 64 && row_tiles / 32 >= 2 * ctas) strides[npass++] = 32;
    strides[npass++] = 1;
    bool have_thr = false;
    B200_CUDA(cudaEventRecord(idx->ev[idx->ev_used], st));
    for (int pi = 0; pi < npass; pi++) {
      const int stride = strides[pi];
      scan_mma_kernel<HILO><<<grid, MS_THREADS, smem, st>>>(tmX, tmQ, n, d, nqb, groups, k, cand, dense, stride,
                                                            have_thr ? thr : nullptr);
      B200_LAUNCH_OK();
      idx->last_scan_launches++;
      if (stride == 1) B200_CUDA(cudaEventRecord(idx->ev[idx->ev_used + 1], st));
      // merge the per-CTA lists: grid*k candidates per query
      B200_TRY(launch_topk_select(dense, M, M, k, C, keys_q, k, 1, nqb, st));
      if (stride > 1) {
        kth_score_kernel<<<(nqb + 255) / 256, 256, 0, st>>>(keys_q, nqb, k, thr);
        B200_LAUNCH_OK();
        have_thr = true;
      }
    }
    idx->ev_used += 2;
  }
  return B200_OK;
}

// max_row ||x||^2 of the scanned table, cached per (pointer, n): one extra read of the table the
// first time a table is scanned in hi-only mode (boot-time cost, 25 ms per 100M x 768 rows).
static int row_norm_bound(b200_index* idx, const __half* rows, int64_t n, float** d_bound, cudaStream_t st) {
  for (int i = 0; i < 2; i++)
    if (idx->norm_rows[i] == rows && idx->norm_n[i] == n && idx->norm_bound[i]) {
      *d_bound = idx->norm_bound[i];
      return B200_OK;
    }
  const int slot = idx->norm_next;
  idx->norm_next ^= 1;
  if (!idx->norm_bound[slot]) B200_CUDA(cudaMalloc(&idx->norm_bound[slot], 256));
  B200_CUDA(cudaMemsetAsync(idx->norm_bound[slot], 0, 4, st));
  row_norm2_max_kernel<<<idx->sms * 8, 256, 0, st>>>(reinterpret_cast<const uint4*>(rows), n, idx->d / 8,
                                                      reinterpret_cast<unsigned int*>(idx->norm_bound[slot]));
  B200_LAUNCH_OK();
  idx->norm_rows[slot] = rows;
  idx->norm_n[slot] = n;
  *d_bound = idx->norm_bound[slot];
  return B200_OK;
}

// Batched scan entry: same contract as scan_topk_keys (knn_scan.cu).
int scan_topk_keys_mma(b200_index* idx, const __half* rows, int64_t n, const float* d_q, int nq, int k,
                       unsigned long long* d_keys_out, cudaStream_t st) {
  const int d = idx->d;
  B200_CHECK(k <= MS_KMAX, B200_ERR_UNSUPPORTED, "mma scan: k=%d > %d", k, MS_KMAX);
  B200_CHECK(n < (1ll << 31), B200_ERR_UNSUPPORTED, "mma scan: at most 2^31 rows per shard");
  // Up to one split-mode group the scan is HBM-bound already; beyond, halve the tensor work.
  const int kc = 2 * k;
  if (!idx->use_hi_only || nq <= MS_QG || kc > MS_KMAX || n < 4 * (int64_t)kc)
    return scan_mma_passes<true>(idx, rows, n, d_q, nq, k, d_keys_out, st);

  float* d_bound = nullptr;
  B200_TRY(row_norm_bound(idx, rows, n, &d_bound, st));
  const size_t al = 255;
  const size_t b_keys = ((size_t)nq * kc * 8 + al) & ~al, b_f = ((size_t)nq * 4 + al) & ~al;
  void* w = nullptr;
  B200_TRY(index_ws(idx, 4, 2 * b_keys + 2 * b_f + 256, &w));
  unsigned long long* approx = (unsigned long long*)w;
  unsigned long long* exact = (unsigned long long*)((char*)w + b_keys);
  float* margin = (float*)((char*)w + 2 * b_keys);
  int* fail_list = (int*)((char*)w + 2 * b_keys + b_f);
  int* fail_count = (int*)((char*)w + 2 * b_keys + 2 * b_f);
  B200_CUDA(cudaMemsetAsync(fail_count, 0, 4, st));
  query_margin_kernel<<<(nq + 7) / 8, 256, 0, st>>>(d_q, nq, d, d_bound, margin);
  B200_LAUNCH_OK();
  B200_TRY(scan_mma_passes<false>(idx, rows, n, d_q, nq, kc, approx, st));
  const int64_t count = (int64_t)nq * kc;
  rescore_kernel<<<(unsigned)((count + 7) / 8), 256, 0, st>>>(reinterpret_cast<const uint4*>(rows), d / 8, d_q, d, approx,
                                                             count, kc, exact);
  B200_LAUNCH_OK();
  int C = 2048;
  while (C < 2 * k) C <<= 1;
  B200_TRY(launch_topk_select(exact, kc, kc, k, C, d_keys_out, k, 1, nq, st));
  verify_kernel<<<(nq + 255) / 256, 256, 0, st>>>(approx, kc, d_keys_out, k, margin, nq, fail_list, fail_count);
  B200_LAUNCH_OK();
  int h_fail = 0;
  B200_CUDA(cudaMemcpyAsync(&h_fail, fail_count, 4, cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  idx->last_hi_only_fallbacks = h_fail;
  if (h_fail > 0) {
    // the proof failed for these queries (candidates packed inside the error bound): split mode
    void* w5 = nullptr;
    const size_t b_q = ((size_t)h_fail * d * 4 + al) & ~al;
    B200_TRY(index_ws(idx, 5, b_q + (size_t)h_fail * k * 8, &w5));
    float* qf = (float*)w5;
    unsigned long long* kf = (unsigned long long*)((char*)w5 + b_q);
    gather_queries_kernel<<<(unsigned)(((int64_t)h_fail * d + 255) / 256), 256, 0, st>>>(d_q, d, fail_list, h_fail, qf);
    B200_LAUNCH_OK();
    B200_TRY(scan_mma_passes<true>(idx, rows, n, qf, h_fail, k, kf, st));
    scatter_keys_kernel<<<(unsigned)(((int64_t)h_fail * k + 255) / 256), 256, 0, st>>>(kf, k, fail_list, h_fail, d_keys_out);
    B200_LAUNCH_OK();
  }
  return B200_OK;
}

}  // namespace b200
