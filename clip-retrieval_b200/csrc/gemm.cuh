// wgmma GEMM core of the embed path (SURVEY.md §2.2 K1, K3, K5, K6, K7):
//   C[M,N] = epilogue(A[M,K] · W[N,K]^T)     A, W bf16 row-major (both "K-major"), fp32 accumulate.
//
// One 128 x BN output tile per CTA, warp-specialised, two CTAs per SM:
//   warp 8      TMA producer: cp.async.bulk.tensor 128x64 (A) and BNx64 (W) boxes, 128B swizzle,
//               into a 3..4-stage shared-memory ring guarded by full/empty mbarriers;
//   warps 0..7  two consumer warpgroups, each issuing wgmma m64nBNk16 over its 64 rows of the tile
//               (fp32 accumulator in registers); a ring slot is released once the wgmma group that
//               read it has completed.  After the k-loop the accumulators go through shared memory
//               (the drained ring) so that the epilogue sees one row per thread: + bias, activation,
//               + residual, bf16 pack, 16-byte global stores.
// Two CTAs per SM let the epilogue of one tile overlap the k-loop of the other.  Tiles are numbered
// in groups of 16 row-blocks x all column-blocks so the activation rows of a group stay in L2 while
// the weights (a few MB) are re-read from L2, not HBM.
// Roofline: tensor pipe; 2*M*N*K flops per launch.
#pragma once
#include "common.cuh"
#include "ptx.cuh"

namespace b200 {

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;
constexpr int GEMM_MMA_K = 16;
constexpr int GEMM_THREADS = 288;  // warps 0..7: two consumer warpgroups (64 rows each), warp 8: TMA producer
constexpr int GEMM_GROUP_M = 16;
constexpr int GEMM_WARP_TMA = 8;

enum { ACT_NONE = 0, ACT_QUICK_GELU = 1, ACT_GELU = 2 };

struct GemmEpilogue {
  const float* bias = nullptr;              // [N] fp32 or null
  const __nv_bfloat16* residual = nullptr;  // added after the activation, or null
  int64_t res_ld = 0;                       // residual leading dimension (elements)
  int res_row_mod = 0;                      // > 0: residual row = res_row_off + row % res_row_mod
  int res_row_off = 0;
  __nv_bfloat16* out = nullptr;
  int64_t out_ld = 0;
  int out_group = 0;                        // > 0: out row = (row / g) * (g + 1) + 1 + row % g  (cls slot)
  int act = ACT_NONE;
  // LayerNorm folded into this GEMM (K5/K6 of SURVEY §2.2 without a separate normalisation pass): A is the RAW
  // residual stream x and the weights carry gamma (W'[n,k] = W[n,k] * gamma[k]), so
  //   LN(x) W^T + b = rstd * (x W'^T - mean * c) + d,   c[n] = sum_k W'[n,k],  d[n] = sum_k beta[k] W[n,k] + b[n].
  // ln_stats: per row, ln_w / 64 records (mean, M2) of 64-column slots of x, written by the producer's epilogue
  // (stats_out below); ln_c = c (fp32 [N]); `bias` then points at d.
  const float2* ln_stats = nullptr;
  const float* ln_c = nullptr;
  int ln_w = 0;
  // Row statistics of what this epilogue stores (bf16-rounded), one (mean, M2) record per 64 output columns:
  // stats_out[row * (N / 64) + slot].  Set on the GEMMs that write the residual stream.
  float2* stats_out = nullptr;
};

// Per-row constants of the epilogue, computed once per tile.
struct EpiRow {
  __nv_bfloat16* out_ptr;
  const __nv_bfloat16* res_ptr;
  float ln_a, ln_b;        // folded LayerNorm: value = acc * ln_a + (ln_b * c[col] + d[col]);  (1, 0) when off
};
// (mean, rstd) of a row from its 64-column slot records (Chan's combination of equal-sized groups).  Every record
// load is issued before the first is used: consuming them one by one pays the L2 latency `slots` times per row.
constexpr int LN_MAX_SLOTS = 24;   // row width <= 1536
__device__ __forceinline__ void ln_row_coeffs(const float2* __restrict__ rec, int slots, int w, float& a, float& b) {
  float2 v[LN_MAX_SLOTS];
#pragma unroll
  for (int i = 0; i < LN_MAX_SLOTS; i++) v[i] = i < slots ? __ldg(rec + i) : make_float2(0.f, 0.f);
  float msum = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_SLOTS; i++) msum += v[i].x;
  const float mean = msum / (float)slots;
  float m2 = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_SLOTS; i++) {
    const float dm = v[i].x - mean;
    m2 += i < slots ? v[i].y + 64.0f * dm * dm : 0.f;
  }
  const float rstd = rsqrtf(fmaxf(m2 / (float)w, 0.f) + 1e-5f);
  a = rstd;
  b = -mean * rstd;
}
__device__ __forceinline__ EpiRow epi_row(const GemmEpilogue& ep, int row, int n0) {
  EpiRow r;
  int64_t out_row = row;
  if (ep.out_group > 0) out_row = (int64_t)(row / ep.out_group) * (ep.out_group + 1) + 1 + row % ep.out_group;
  int64_t res_row = row;
  if (ep.res_row_mod > 0) res_row = ep.res_row_off + row % ep.res_row_mod;
  r.out_ptr = ep.out + out_row * ep.out_ld + n0;
  r.res_ptr = ep.residual ? ep.residual + res_row * ep.res_ld + n0 : nullptr;
  r.ln_a = 1.0f;
  r.ln_b = 0.0f;
  return r;
}

template <int BN>
struct GemmCfg {
  static_assert(BN == 32 || BN == 64 || BN == 128, "tile widths: 32, 64, 128");
  // narrow tiles (BN = 64 / 32) exist for the serving shapes: with M <= 128 rows a GEMM has N / BN tiles in total, and
  // the weight read (the whole cost at batch 1) is spread over that many SMs.  The ring stays under ~100 KB so that two
  // CTAs share an SM.
  static constexpr int STAGES = BN == 128 ? 3 : 4;
  static constexpr int A_BYTES = GEMM_BM * GEMM_BK * 2;
  static constexpr int B_BYTES = BN * GEMM_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int RING_BYTES = STAGES * STAGE_BYTES;
  static constexpr int STG_LD = BN + 4;   // fp32 staging row pitch (floats): conflict-free 16-byte row reads
  static_assert(GEMM_BM * STG_LD * 4 <= RING_BYTES, "the accumulator staging tile reuses the ring");
  static constexpr int SMEM_BYTES = RING_BYTES + 2 * BN * 4 + 256 + 1024;  // ring + bias + LN c + barriers + align slack
};

__device__ __forceinline__ void gemm_tile_coords(int tile, int mb, int nb, int& m_blk, int& n_blk) {
  const int per_group = GEMM_GROUP_M * nb;
  const int g = tile / per_group;
  const int first_m = g * GEMM_GROUP_M;
  const int gsize = min(GEMM_GROUP_M, mb - first_m);
  const int r = tile - g * per_group;
  m_blk = first_m + r % gsize;
  n_blk = r / gsize;
}

__device__ __forceinline__ float act_apply(float x, int act) {
  if (act == ACT_QUICK_GELU) {
    // x * sigmoid(1.702 x), sigmoid(y) = 0.5 * tanh(y / 2) + 0.5: one MUFU op per element
    float t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.851f * x));
    return x * fmaf(0.5f, t, 0.5f);
  } else if (act == ACT_GELU) {
    return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f));
  }
  return x;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}

// bias + activation + residual + bf16 store of 8 consecutive columns (col = offset inside the tile)
// `rr` = the residual's 8 values, loaded before the accumulator is read so that their HBM latency does not sit in
// the middle of the epilogue.
// s_bias = bias (or the folded LayerNorm's d), s_c = the folded LayerNorm's c (read only when ep.ln_stats is set).
// st_k / st_s / st_q: running shifted sums of the stored values for the row statistics (ep.stats_out).
// SPEC: -1 = every feature decided at run time; 0..7 = activation | residual << 2 fixed at compile time (no LayerNorm
// fold, no row statistics): the generic flavour carries a run-time activation switch around an inlined
// erff for every element plus the fold / statistics paths.
template <int SPEC>
__device__ __forceinline__ void epi_store8(const GemmEpilogue& ep, const EpiRow& er, const uint32_t* r8,
                                           const float* s_bias, const float* s_c, int col, int n0, const uint4& rr,
                                           float st_k, float& st_s, float& st_q) {
  const int act = SPEC >= 0 ? (SPEC & 3) : ep.act;
  const bool use_ln = SPEC < 0 && ep.ln_stats != nullptr;
  const bool use_stats = SPEC < 0 && ep.stats_out != nullptr;
  const bool has_res = SPEC >= 0 ? ((SPEC >> 2) & 1) != 0 : er.res_ptr != nullptr;
  float v[8];
  if (use_ln) {
#pragma unroll
    for (int j = 0; j < 8; j++)
      v[j] = act_apply(fmaf(__uint_as_float(r8[j]), er.ln_a, fmaf(er.ln_b, s_c[col + j], s_bias[col + j])), act);
  } else {
#pragma unroll
    for (int j = 0; j < 8; j++) v[j] = act_apply(__uint_as_float(r8[j]) + s_bias[col + j], act);
  }
  if (has_res) {
    const float2 a = unpack_bf16x2(rr.x), b = unpack_bf16x2(rr.y), cc = unpack_bf16x2(rr.z), dd = unpack_bf16x2(rr.w);
    // __fadd_rn: never contracted with the activation's last multiply into an FMA — every epilogue flavour (run-time or
    // compile-time) rounds the same way and stays bit-identical to the others
    v[0] = __fadd_rn(v[0], a.x); v[1] = __fadd_rn(v[1], a.y); v[2] = __fadd_rn(v[2], b.x); v[3] = __fadd_rn(v[3], b.y);
    v[4] = __fadd_rn(v[4], cc.x); v[5] = __fadd_rn(v[5], cc.y); v[6] = __fadd_rn(v[6], dd.x); v[7] = __fadd_rn(v[7], dd.y);
  }
  uint4 o;
  o.x = pack_bf16x2(v[0], v[1]);
  o.y = pack_bf16x2(v[2], v[3]);
  o.z = pack_bf16x2(v[4], v[5]);
  o.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(er.out_ptr + col) = o;
  if (use_stats) {
    // statistics of the values as stored (bf16), shifted by the slot's first value to keep the sums small
    const float2 f0 = unpack_bf16x2(o.x), f1 = unpack_bf16x2(o.y), f2 = unpack_bf16x2(o.z), f3 = unpack_bf16x2(o.w);
    const float e[8] = {f0.x - st_k, f0.y - st_k, f1.x - st_k, f1.y - st_k, f2.x - st_k, f2.y - st_k, f3.x - st_k, f3.y - st_k};
#pragma unroll
    for (int j = 0; j < 8; j++) {
      st_s += e[j];
      st_q = fmaf(e[j], e[j], st_q);
    }
  }
}

// One 32-column chunk `c` of the tile for this thread's row: the four 8-column groups, and (stats_out) the
// (mean, M2) record of a completed 64-column slot (chunks 2j, 2j+1).
template <int SPEC>
__device__ __forceinline__ void epi_chunk(const GemmEpilogue& ep, const EpiRow& er, const uint32_t* r, const float* s_bias,
                                          const float* s_c, int c, int n0, int N, int row, const uint4* res4, float& st_k,
                                          float& st_s, float& st_q) {
  const bool use_stats = SPEC < 0 && ep.stats_out != nullptr;
  if (use_stats && (c & 1) == 0) {
    // shift = what the first column of the slot will store (bf16): recomputed here, cheap
    st_s = 0.f;
    st_q = 0.f;
    float v0;
    const int col = c * 32;
    if (ep.ln_stats != nullptr) v0 = act_apply(fmaf(__uint_as_float(r[0]), er.ln_a, fmaf(er.ln_b, s_c[col], s_bias[col])), ep.act);
    else v0 = act_apply(__uint_as_float(r[0]) + s_bias[col], ep.act);
    if (er.res_ptr) v0 = __fadd_rn(v0, unpack_bf16x2(res4[0].x).x);
    st_k = __bfloat162float(__float2bfloat16_rn(v0));
  }
#pragma unroll
  for (int g = 0; g < 4; g++) {
    const int col = c * 32 + g * 8;
    if (n0 + col < N) epi_store8<SPEC>(ep, er, r + g * 8, s_bias, s_c, col, n0, res4[g], st_k, st_s, st_q);
  }
  if (use_stats && (c & 1) == 1 && n0 + c * 32 < N) {
    const float mean = st_k + st_s * (1.0f / 64.0f);
    const float m2 = fmaxf(st_q - st_s * st_s * (1.0f / 64.0f), 0.f);
    ep.stats_out[(int64_t)row * (N >> 6) + ((n0 + c * 32) >> 6)] = make_float2(mean, m2);
  }
}

template <int BN, int SPEC = -1>
__global__ void __launch_bounds__(GEMM_THREADS, 2)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, int M, int N,
                       int K, GemmEpilogue ep) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = ptx::smem_u32(smem_raw);
  uint8_t* base = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* sA = base;
  uint8_t* sB = base + STAGES * Cfg::A_BYTES;
  float* s_bias = reinterpret_cast<float*>(base + Cfg::RING_BYTES);
  float* s_c = s_bias + BN;
  uint64_t* full = reinterpret_cast<uint64_t*>(s_c + BN);
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int mb = (M + GEMM_BM - 1) / GEMM_BM, nb = (N + BN - 1) / BN, kb = (K + GEMM_BK - 1) / GEMM_BK;
  int m_blk, n_blk;
  gemm_tile_coords(blockIdx.x, mb, nb, m_blk, n_blk);
  const int n0 = n_blk * BN;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; s++) {
      ptx::mbar_init(&full[s], 1);
      ptx::mbar_init(&empty[s], 8);  // one arrive per consumer warp
    }
    ptx::fence_barrier_init();
  }
  for (int j = threadIdx.x; j < BN; j += GEMM_THREADS) {
    s_bias[j] = (ep.bias != nullptr && n0 + j < N) ? ep.bias[n0 + j] : 0.0f;
    if (SPEC < 0) s_c[j] = (ep.ln_c != nullptr && n0 + j < N) ? ep.ln_c[n0 + j] : 0.0f;
  }
  __syncthreads();

  if (warp == GEMM_WARP_TMA) {
    // ---------------- TMA producer ----------------
    if (lane == 0) {
      ptx::prefetch_tensormap(&tmA);
      ptx::prefetch_tensormap(&tmB);
      for (int kbi = 0; kbi < kb; kbi++) {
        const int stage = kbi % STAGES;
        if (kbi >= STAGES) ptx::mbar_wait(&empty[stage], ((kbi / STAGES) - 1) & 1);
        ptx::mbar_arrive_expect_tx(&full[stage], Cfg::STAGE_BYTES);
        ptx::tma_load_2d(sA + stage * Cfg::A_BYTES, &tmA, &full[stage], kbi * GEMM_BK, m_blk * GEMM_BM);
        ptx::tma_load_2d(sB + stage * Cfg::B_BYTES, &tmB, &full[stage], kbi * GEMM_BK, n0);
      }
    }
    return;
  }

  // ---------------- consumers (warps 0..7): wgmma main loop ----------------
  const int wg = warp >> 2;   // rows wg*64 .. wg*64+63 of the tile
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; i++) acc[i] = 0.f;
  for (int kbi = 0; kbi < kb; kbi++) {
    const int stage = kbi % STAGES;
    ptx::mbar_wait(&full[stage], (kbi / STAGES) & 1);
    ptx::wgmma_fence();
    const uint64_t da = ptx::wgmma_desc_k_sw128(ptx::smem_u32(sA + stage * Cfg::A_BYTES + wg * 64 * 128));
    const uint64_t db = ptx::wgmma_desc_k_sw128(ptx::smem_u32(sB + stage * Cfg::B_BYTES));
#pragma unroll
    for (int k = 0; k < GEMM_BK / GEMM_MMA_K; k++)
      ptx::wgmma_bf16<BN>(acc, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (kbi | k) != 0 ? 1u : 0u);
    ptx::wgmma_commit();
    // the group of the previous k-block has completed: its ring slot may be refilled
    ptx::wgmma_wait<1>();
    if (kbi > 0 && lane == 0) ptx::mbar_arrive(&empty[(kbi - 1) % STAGES]);
  }
  ptx::wgmma_wait<0>();
  ptx::fence_regs(acc);

  // ---------------- epilogue ----------------
  // every load has landed and every wgmma has read its operands: the ring becomes the fp32 staging tile
  float* stg = reinterpret_cast<float*>(base);
  ptx::fence_proxy_async();
  asm volatile("bar.sync 1, 256;" ::: "memory");
  {
    const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; j++) {
      *reinterpret_cast<float2*>(stg + r * Cfg::STG_LD + 8 * j + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(stg + (r + 8) * Cfg::STG_LD + 8 * j + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");

  const int q = warp & 3;            // 32-row quarter of the tile
  const int half = warp >> 2;        // which half of the tile columns this warp drains
  const int lrow = q * 32 + lane;
  const int row = m_blk * GEMM_BM + lrow;
  const bool row_ok = row < M;
  constexpr int CPW = BN >= 64 ? BN / 64 : 1;   // 32-column chunks per epilogue warp
  if (!row_ok || half * CPW * 32 >= BN) return;  // BN = 32: the second warp of each quarter has no columns
  EpiRow er = epi_row(ep, row, n0);
  if (SPEC < 0 && ep.ln_stats != nullptr) ln_row_coeffs(ep.ln_stats + (int64_t)row * (ep.ln_w >> 6), ep.ln_w >> 6, ep.ln_w, er.ln_a, er.ln_b);
  float st_k = 0.f, st_s = 0.f, st_q = 0.f;
  uint4 res[CPW][4];
#pragma unroll
  for (int ci = 0; ci < CPW; ci++) {
#pragma unroll
    for (int g = 0; g < 4; g++) {
      const int col = (half * CPW + ci) * 32 + g * 8;
      const bool want = SPEC >= 0 ? ((SPEC >> 2) & 1) != 0 : er.res_ptr != nullptr;
      res[ci][g] = (want && n0 + col < N) ? *reinterpret_cast<const uint4*>(er.res_ptr + col) : make_uint4(0u, 0u, 0u, 0u);
    }
  }
#pragma unroll
  for (int ci = 0; ci < CPW; ci++) {
    const int c = half * CPW + ci;
    uint32_t r[32];
    const float4* src4 = reinterpret_cast<const float4*>(stg + lrow * Cfg::STG_LD + c * 32);
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const float4 v = src4[i];
      r[4 * i] = __float_as_uint(v.x); r[4 * i + 1] = __float_as_uint(v.y);
      r[4 * i + 2] = __float_as_uint(v.z); r[4 * i + 3] = __float_as_uint(v.w);
    }
    epi_chunk<SPEC>(ep, er, r, s_bias, s_c, c, n0, N, row, res[ci], st_k, st_s, st_q);
  }
}

// host side (gemm.cu)
int make_tmap_2d(CUtensorMap* out, const void* ptr, int dtype_bf16, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                 uint32_t box_rows, uint32_t box_cols);
// tmB must have boxes of bn rows x 64 columns.
int gemm_bf16_launch(const CUtensorMap& tmA, const CUtensorMap& tmB, int bn, int M, int N, int K,
                     const GemmEpilogue& ep, cudaStream_t st);
// Pick the column-block width for a GEMM with N output columns (128, or 64 / 32 when the grid would be
// under-filled).
int gemm_pick_bn(int M, int N, int sms);

}  // namespace b200
