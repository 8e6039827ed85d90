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

// ACT_RELU is internal (the ResNet image tower): relu(acc + bias + residual), the residual added *before* the
// activation.  The public GEMM entries accept 0..2 only.
enum { ACT_NONE = 0, ACT_QUICK_GELU = 1, ACT_GELU = 2, ACT_RELU = 3 };

struct GemmEpilogue {
  const float* bias = nullptr;              // [N] fp32 or null
  const __nv_bfloat16* residual = nullptr;  // added after the activation (before it for ACT_RELU), or null
  int64_t res_ld = 0;                       // residual leading dimension (elements)
  int res_row_mod = 0;                      // > 0: residual row = res_row_off + row % res_row_mod
  int res_row_off = 0;
  __nv_bfloat16* out = nullptr;
  int64_t out_ld = 0;
  int out_group = 0;                        // > 0: out row = (row / g) * (g + 1) + 1 + row % g  (cls slot)
  int act = ACT_NONE;
};

// Per-row constants of the epilogue, computed once per tile.
struct EpiRow {
  __nv_bfloat16* out_ptr;
  const __nv_bfloat16* res_ptr;
};
__device__ __forceinline__ EpiRow epi_row(const GemmEpilogue& ep, int row, int n0) {
  EpiRow r;
  int64_t out_row = row;
  if (ep.out_group > 0) out_row = (int64_t)(row / ep.out_group) * (ep.out_group + 1) + 1 + row % ep.out_group;
  int64_t res_row = row;
  if (ep.res_row_mod > 0) res_row = ep.res_row_off + row % ep.res_row_mod;
  r.out_ptr = ep.out + out_row * ep.out_ld + n0;
  r.res_ptr = ep.residual ? ep.residual + res_row * ep.res_ld + n0 : nullptr;
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
  static constexpr int SMEM_BYTES = RING_BYTES + BN * 4 + 256 + 1024;  // ring + bias + barriers + align slack
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

// act(pre) + residual, pre = accumulator + bias: the per-element arithmetic of every epilogue, rounded to bf16 by the
// caller (pack_bf16x2).  __fadd_rn: never contracted with the activation's last multiply into an FMA — every epilogue
// (either kernel, register or TMA store) rounds the same way and stays bit-identical to the others.
// ACT_RELU: relu(pre + residual), the bottleneck block's `out += identity; out = relu(out)`.
__device__ __forceinline__ float epi_apply(float pre, int act, bool has_res, float res) {
  if (act == ACT_RELU) return fmaxf(has_res ? __fadd_rn(pre, res) : pre, 0.0f);
  const float v = act_apply(pre, act);
  return has_res ? __fadd_rn(v, res) : v;
}

// bias + activation + residual + bf16 store of 8 consecutive columns (col = offset inside the tile)
// `rr` = the residual's 8 values, loaded before the accumulator is read so that their HBM latency does not sit in
// the middle of the epilogue.
// SPEC = activation | residual << 2, fixed at compile time.
template <int SPEC>
__device__ __forceinline__ void epi_store8(const EpiRow& er, const uint32_t* r8, const float* s_bias, int col,
                                           const uint4& rr) {
  constexpr int act = SPEC & 3;
  constexpr bool has_res = ((SPEC >> 2) & 1) != 0;
  const float2 a = unpack_bf16x2(rr.x), b = unpack_bf16x2(rr.y), cc = unpack_bf16x2(rr.z), dd = unpack_bf16x2(rr.w);
  const float res[8] = {a.x, a.y, b.x, b.y, cc.x, cc.y, dd.x, dd.y};
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; j++) v[j] = epi_apply(__uint_as_float(r8[j]) + s_bias[col + j], act, has_res, res[j]);
  uint4 o;
  o.x = pack_bf16x2(v[0], v[1]);
  o.y = pack_bf16x2(v[2], v[3]);
  o.z = pack_bf16x2(v[4], v[5]);
  o.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(er.out_ptr + col) = o;
}

// One 32-column chunk `c` of the tile for this thread's row: the four 8-column groups.
template <int SPEC>
__device__ __forceinline__ void epi_chunk(const EpiRow& er, const uint32_t* r, const float* s_bias, int c, int n0, int N,
                                          const uint4* res4) {
#pragma unroll
  for (int g = 0; g < 4; g++) {
    const int col = c * 32 + g * 8;
    if (n0 + col < N) epi_store8<SPEC>(er, r + g * 8, s_bias, col, res4[g]);
  }
}

// Geometry of an implicit 3x3 stride-1 pad-1 convolution (conv.cu): the A operand is the NHWC activation [B, H, W, C]
// read through an im2col tensor map, K = 9 * cb * 64 with k-block kbi = tap * cb + channel slice, tap = 3 r + s.
struct ConvGeom {
  int H = 0, W = 0, cb = 0;   // cb = ceil(C / 64)
};

// The 128-row tile of one CTA.  CONV: the producer's A box is one im2col load (128 output pixels x 64 channels of one
// tap, borders and channels >= C zero-filled by TMA) instead of a 128 x 64 tile of A; everything else is shared.
template <int BN, int SPEC, bool CONV>
__device__ __forceinline__ void gemm_bf16_wgmma_tile(const CUtensorMap& tmA, const CUtensorMap& tmB, int M, int N, int K,
                                                     const GemmEpilogue& ep, const ConvGeom& cg) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = ptx::smem_u32(smem_raw);
  uint8_t* base = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* sA = base;
  uint8_t* sB = base + STAGES * Cfg::A_BYTES;
  float* s_bias = reinterpret_cast<float*>(base + Cfg::RING_BYTES);
  uint64_t* full = reinterpret_cast<uint64_t*>(s_bias + BN);
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
  for (int j = threadIdx.x; j < BN; j += GEMM_THREADS)
    s_bias[j] = (ep.bias != nullptr && n0 + j < N) ? ep.bias[n0 + j] : 0.0f;
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
        if constexpr (CONV) {
          // output pixel m_blk * 128 = (n, h, w): the box starts at input pixel (h - 1, w - 1) of image n, the tap's
          // (r, s) offset is added to every pixel of it; rows run on across image rows and images
          const int tap = kbi / cg.cb, cs = kbi - tap * cg.cb;
          const int m0 = m_blk * GEMM_BM, hw = cg.H * cg.W;
          const int n = m0 / hw, rem = m0 - n * hw, h = rem / cg.W, w = rem - h * cg.W;
          ptx::tma_load_im2col_4d(sA + stage * Cfg::A_BYTES, &tmA, &full[stage], cs * GEMM_BK, w - 1, h - 1, n,
                                  (uint16_t)(tap % 3), (uint16_t)(tap / 3));
        } else {
          ptx::tma_load_2d(sA + stage * Cfg::A_BYTES, &tmA, &full[stage], kbi * GEMM_BK, m_blk * GEMM_BM);
        }
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
  const EpiRow er = epi_row(ep, row, n0);
  uint4 res[CPW][4];
#pragma unroll
  for (int ci = 0; ci < CPW; ci++) {
#pragma unroll
    for (int g = 0; g < 4; g++) {
      const int col = (half * CPW + ci) * 32 + g * 8;
      constexpr bool want = ((SPEC >> 2) & 1) != 0;
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
    epi_chunk<SPEC>(er, r, s_bias, c, n0, N, res[ci]);
  }
}

template <int BN, int SPEC>
__global__ void __launch_bounds__(GEMM_THREADS, 2)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, int M, int N,
                       int K, GemmEpilogue ep) {
  gemm_bf16_wgmma_tile<BN, SPEC, false>(tmA, tmB, M, N, K, ep, ConvGeom());
}

// Implicit-GEMM 3x3 convolution (stride 1, pad 1): out[B*H*W, N] = epilogue(im2col(x) · W^T), W packed [N, 9 * cb * 64]
// (conv.cu).  tmA is an im2col map over x [B, H, W, C] (make_tmap_im2col_3x3).
template <int BN, int SPEC>
__global__ void __launch_bounds__(GEMM_THREADS, 2)
conv3x3_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, int M, int N,
                          int K, GemmEpilogue ep, ConvGeom cg) {
  gemm_bf16_wgmma_tile<BN, SPEC, true>(tmA, tmB, M, N, K, ep, cg);
}

// ---- persistent 128 x 256 tiles for the large-batch shapes ----------------------------------------------------
// One CTA per SM (384 threads) loops over the tiles blockIdx.x, blockIdx.x + gridDim.x, ... in gemm_tile_coords' order:
//   warpgroup 0     thread 0, the k-block producer (its registers go to the consumers): a 128x64 A box and two
//                   128x64 W boxes per k-block into a ring of 48 KB stages.  It runs on into the next tile's k-blocks
//                   while the consumers are in the epilogue of this one.
//                   thread 32, the staging thread (TMA-store epilogue): loads the residual boxes of a tile into the
//                   bf16 staging tile while the consumers are still in its k-loop, stores the finished tile by TMA, and
//                   hands the staging tile back once those stores have read it.
//   warpgroups 1-2  consumers, each issuing wgmma m64n256k16 over its 64 rows of the tile (128 fp32 accumulators per
//                   thread).  Per 64-deep k-block a CTA loads 48 KB for 1024 tensor-pipe clocks of math, against 32 KB
//                   for 512 at 128 x 128: a third less L2 -> SM traffic per flop.
// Epilogue (TMA store, every GEMM without a row map): each consumer converts its accumulators in fragment layout,
// act(acc + bias) + residual (epi_apply), and writes bf16 pairs into its warpgroup's half of the staging tile, four
// 64 x 64 boxes in the 128B-swizzled layout of the output tensor map (the residual, loaded there by TMA, is read from
// and overwritten in place).  Then fence.proxy.async, one arrive per thread on the warpgroup's stg_full barrier, and
// straight on into the next tile's k-loop: the staging thread issues the TMA stores, which drain behind that k-loop, and
// the consumers wait for the staging tile (stg_ready) only at their next epilogue.  The premise: every CTA reaches
// its epilogues at about the same moment, so stores from registers stall all SMs at once behind a burst of 8.6 MB
// (17 MB with the residual read).  Measured (tools/gemm_bench.py --ksweep, DESIGN.md §8): the fixed cost per tile fell
// by half or more for the plain and GELU epilogues, and less with a residual; the rest is the consumers' conversion work.
// The TMA-store epilogue is taken from 8 tiles per CTA up (gemm.cu): below that its 3-stage ring costs more than the
// overlap saves.
// Row maps (out_group / res_row_mod: the patch embedding, one GEMM per image tower) and small grids keep a
// register-store epilogue with a 4-stage ring:
// each warp passes its 16 x 256 slab through a private 16 x 32 fp32 staging chunk so that its stores run along rows.
// Both epilogues compute every element with epi_apply, so outputs are bit-identical to the 128-wide kernel's (the
// same k16 wgmma sequence feeds it).
// A variant with CTA pairs (clusters of 2 along M) multicasting one 128-row W half each was built and measured slower
// at every bench shape (DESIGN.md §8), so W is loaded per CTA.
constexpr int GEMM_WIDE_BN = 256;
constexpr int GEMM_WIDE_THREADS = 384;
constexpr int GEMM_WIDE_BOX = 64;   // rows and columns of a TMA box of the output / residual maps (128 bytes per row)
// STAGES_: ring depth.  STG_BOXES_: 64-column boxes of each warpgroup's 64 rows in the bf16 staging tile (4: the whole
// 128 x 256 tile; 2: half of it, staged and stored in two passes per tile), or 0 for the register-store epilogue.
template <int STAGES_, int STG_BOXES_>
struct GemmWideCfg {
  static constexpr int STAGES = STAGES_;
  static constexpr int STG_BOXES = STG_BOXES_;
  static constexpr int A_BYTES = GEMM_BM * GEMM_BK * 2;        // 16 KB
  static constexpr int B_BYTES = GEMM_WIDE_BN * GEMM_BK * 2;   // 32 KB: two 128-row W boxes
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int RING_BYTES = STAGES * STAGE_BYTES;
  static constexpr int BOX_BYTES = GEMM_WIDE_BOX * GEMM_WIDE_BOX * 2;   // 8 KB, 1024-byte aligned (the swizzle atom)
  static constexpr int STG_LD = 40;   // register-store epilogue: fp32 chunk pitch (floats), conflict-free float2 writes
                                      // and (with the odd-row order below) float4 reads
  static constexpr int STG_BYTES = STG_BOXES > 0 ? 2 * STG_BOXES * BOX_BYTES     // two warpgroups' boxes
                                                 : 8 * 16 * STG_LD * 4;           // 8 consumer warps x 16 x 32 fp32
  static constexpr int PASSES = STG_BOXES > 0 ? 4 / STG_BOXES : 1;   // staging passes per tile
  // Two bias rows (alternate tiles, so one tile's epilogue never races the next fill) where they fit; the half-tile
  // variant with its 4-stage ring has room for one, refilled behind a barrier.
  static constexpr int BIAS_ROWS = STG_BOXES == 2 ? 1 : 2;
  // + bias rows, 16 mbarriers, and the slack to align the ring to 1024 bytes
  static constexpr int SMEM_BYTES = RING_BYTES + STG_BYTES + BIAS_ROWS * GEMM_WIDE_BN * 4 + 128 + 1024;
  // STG_BOXES = 2 (4-stage ring, half a tile in two passes) fits in 231 552 B but failed a bit-identity check at
  // M = 1, N = 264 when first run, and is not used (DESIGN.md §8)
  static_assert(STG_BOXES == 0 || STG_BOXES == 4, "the staging tile holds a whole tile");
  static_assert(SMEM_BYTES <= 227 * 1024, "the persistent GEMM's shared memory exceeds an SM's");
};
using GemmWideTmaCfg = GemmWideCfg<3, 4>;       // 144 KB ring + 64 KB staging tile
using GemmWideRegCfg = GemmWideCfg<4, 0>;       // 192 KB ring + 20 KB of fp32 chunks

template <int SPEC, class Cfg>
__global__ void __launch_bounds__(GEMM_WIDE_THREADS, 1)
gemm_bf16_wgmma_persistent_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                                  const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmR,
                                  int M, int N, int K, GemmEpilogue ep) {
  constexpr int STAGES = Cfg::STAGES;
  constexpr int BN = GEMM_WIDE_BN;
  constexpr bool HAS_RES = ((SPEC >> 2) & 1) != 0;
  constexpr bool TMA_EPI = Cfg::STG_BOXES > 0;   // tmC (and with a residual tmR) are read only then
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = ptx::smem_u32(smem_raw);
  uint8_t* base = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* sA = base;
  uint8_t* sB = base + STAGES * Cfg::A_BYTES;
  uint8_t* s_stg = base + Cfg::RING_BYTES;         // 1024-byte aligned: RING_BYTES is a multiple of 16 KB
  float* s_bias = reinterpret_cast<float*>(s_stg + Cfg::STG_BYTES);   // [BIAS_ROWS][BN]
  uint64_t* full = reinterpret_cast<uint64_t*>(s_bias + Cfg::BIAS_ROWS * BN);
  uint64_t* empty = full + STAGES;
  uint64_t* stg_ready = empty + STAGES;   // [2] per warpgroup: its staging boxes may be written (residual landed)
  uint64_t* stg_full = stg_ready + 2;     // [2] per warpgroup: its staging boxes hold the finished tile

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int mb = (M + GEMM_BM - 1) / GEMM_BM, nb = (N + BN - 1) / BN, kb = (K + GEMM_BK - 1) / GEMM_BK;
  const int tiles = mb * nb;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; s++) {
      ptx::mbar_init(&full[s], 1);
      ptx::mbar_init(&empty[s], 8);  // one arrive per consumer warp
    }
    for (int g = 0; g < 2; g++) {
      ptx::mbar_init(&stg_ready[g], 1);
      ptx::mbar_init(&stg_full[g], 128);   // every thread of the warpgroup, after its fence.proxy.async
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    ptx::setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      // ---------------- TMA producer ----------------
      ptx::prefetch_tensormap(&tmA);
      ptx::prefetch_tensormap(&tmB);
      int it = 0;   // k-blocks issued by this CTA over all its tiles: the ring position
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        int m_blk, n_blk;
        gemm_tile_coords(tile, mb, nb, m_blk, n_blk);
        for (int kbi = 0; kbi < kb; kbi++, it++) {
          const int stage = it % STAGES;
          if (it >= STAGES) ptx::mbar_wait(&empty[stage], ((it / STAGES) - 1) & 1);
          ptx::mbar_arrive_expect_tx(&full[stage], Cfg::STAGE_BYTES);
          uint8_t* b = sB + stage * Cfg::B_BYTES;
          ptx::tma_load_2d(sA + stage * Cfg::A_BYTES, &tmA, &full[stage], kbi * GEMM_BK, m_blk * GEMM_BM);
          ptx::tma_load_2d(b, &tmB, &full[stage], kbi * GEMM_BK, n_blk * BN);
          ptx::tma_load_2d(b + Cfg::B_BYTES / 2, &tmB, &full[stage], kbi * GEMM_BK, n_blk * BN + 128);
        }
      }
    } else if (TMA_EPI && threadIdx.x == 32) {
      // ---------------- staging thread: residual loads and output stores ----------------
      ptx::prefetch_tensormap(&tmC);
      if (HAS_RES) ptx::prefetch_tensormap(&tmR);
      // Boxes of warpgroup g in staging pass `pass` of `tile` that lie inside M and N (the others are neither loaded
      // nor stored): the first one covers columns c0 + pass * STG_BOXES * 64.
      auto live_boxes = [&](int m_blk, int c0, int pass, int g) {
        if (m_blk * GEMM_BM + g * GEMM_WIDE_BOX >= M) return 0;
        return max(0, min(Cfg::STG_BOXES, (N - c0 + GEMM_WIDE_BOX - 1) / GEMM_WIDE_BOX - pass * Cfg::STG_BOXES));
      };
      // Hands warpgroup g's staging boxes to its consumers for a pass: with the residual loaded into them, else at once.
      auto open = [&](int tile, int pass, int g) {
        if (tile >= tiles) return;
        if (!HAS_RES) {
          ptx::mbar_arrive(&stg_ready[g]);
          return;
        }
        int m_blk, n_blk;
        gemm_tile_coords(tile, mb, nb, m_blk, n_blk);
        const int boxes = live_boxes(m_blk, n_blk * BN, pass, g);
        ptx::mbar_arrive_expect_tx(&stg_ready[g], boxes * Cfg::BOX_BYTES);
        for (int b = 0; b < boxes; b++)
          ptx::tma_load_2d(s_stg + (g * Cfg::STG_BOXES + b) * Cfg::BOX_BYTES, &tmR, &stg_ready[g],
                           n_blk * BN + (pass * Cfg::STG_BOXES + b) * GEMM_WIDE_BOX, m_blk * GEMM_BM + g * GEMM_WIDE_BOX);
      };
      open(blockIdx.x, 0, 0);
      open(blockIdx.x, 0, 1);
      int ph = 0;   // staging passes completed: the phase of stg_full
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        int m_blk, n_blk;
        gemm_tile_coords(tile, mb, nb, m_blk, n_blk);
        const int c0 = n_blk * BN;
        for (int pass = 0; pass < Cfg::PASSES; pass++, ph++) {
          for (int g = 0; g < 2; g++) {
            ptx::mbar_wait(&stg_full[g], ph & 1);
            const int boxes = live_boxes(m_blk, c0, pass, g);
            for (int b = 0; b < boxes; b++)
              ptx::tma_store_2d(&tmC, s_stg + (g * Cfg::STG_BOXES + b) * Cfg::BOX_BYTES,
                                c0 + (pass * Cfg::STG_BOXES + b) * GEMM_WIDE_BOX, m_blk * GEMM_BM + g * GEMM_WIDE_BOX);
            ptx::bulk_commit_group();
          }
          // once the stores have read a warpgroup's boxes, they take the next pass's residual
          const int next_tile = pass + 1 < Cfg::PASSES ? tile : tile + gridDim.x;
          const int next_pass = pass + 1 < Cfg::PASSES ? pass + 1 : 0;
          ptx::bulk_wait_group_read<1>();
          open(next_tile, next_pass, 0);
          ptx::bulk_wait_group_read<0>();
          open(next_tile, next_pass, 1);
        }
      }
      ptx::bulk_wait_group<0>();
    }
    return;
  }

  // ---------------- consumers (warps 4..11) ----------------
  ptx::setmaxnreg_inc<232>();
  const int cw = warp - 4;                  // consumer warp 0..7
  const int wg = cw >> 2;                   // rows wg*64 .. wg*64+63 of the tile
  const int ct = threadIdx.x - 128;         // 0..255
  const int fr = lane >> 2, fc = lane & 3;  // accumulator fragment: rows fr, fr + 8 of the warp's 16; columns 8 j + 2 fc
  float acc[BN / 2];
  int it = 0;
  for (int tile = blockIdx.x, local = 0; tile < tiles; tile += gridDim.x, local++) {
    int m_blk, n_blk;
    gemm_tile_coords(tile, mb, nb, m_blk, n_blk);
    const int n0 = n_blk * BN;
    float* bias_t = s_bias + (local % Cfg::BIAS_ROWS) * BN;
    if (Cfg::BIAS_ROWS == 1 && local > 0) ptx::named_barrier_sync(1, 256);   // the last tile's epilogue has read it
    bias_t[ct] = (ep.bias != nullptr && n0 + ct < N) ? ep.bias[n0 + ct] : 0.0f;
    if (HAS_RES && !TMA_EPI) {
      // the residual rows of the tile are brought to L2 while the k-loop runs (two 128-byte lines per thread)
      const int row = m_blk * GEMM_BM + (ct >> 1);
      const int col = (ct & 1) * 128;
      if (row < M) {
        const EpiRow er = epi_row(ep, row, n0);
        if (n0 + col < N) ptx::prefetch_l2(er.res_ptr + col);
        if (n0 + col + 64 < N) ptx::prefetch_l2(er.res_ptr + col + 64);
      }
    }
    ptx::named_barrier_sync(1, 256);   // bias_t is filled

    for (int kbi = 0; kbi < kb; kbi++, it++) {
      const int stage = it % STAGES;
      ptx::mbar_wait(&full[stage], (it / STAGES) & 1);
      ptx::wgmma_fence();
      const uint64_t da = ptx::wgmma_desc_k_sw128(ptx::smem_u32(sA + stage * Cfg::A_BYTES + wg * 64 * 128));
      const uint64_t db = ptx::wgmma_desc_k_sw128(ptx::smem_u32(sB + stage * Cfg::B_BYTES));
#pragma unroll
      for (int k = 0; k < GEMM_BK / GEMM_MMA_K; k++)
        ptx::wgmma_bf16<BN>(acc, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (kbi | k) != 0 ? 1u : 0u);
      ptx::wgmma_commit();
      // the group of the previous k-block has completed: its ring slot may be refilled
      ptx::wgmma_wait<1>();
      if (kbi > 0 && lane == 0) ptx::mbar_arrive(&empty[(it - 1) % STAGES]);
    }
    ptx::wgmma_wait<0>();
    ptx::fence_regs(acc);
    if (lane == 0) ptx::mbar_arrive(&empty[(it - 1) % STAGES]);

    if constexpr (TMA_EPI) {
      // ---------------- epilogue: fragments into the swizzled staging boxes, stored by the staging thread ----------
      // Row r of a box is 128 bytes; its 16-byte chunk q lies at chunk q ^ (r % 8) (128B swizzle).  Lane (fr, fc)
      // writes columns 8 j + 2 fc, +1 of rows fr and fr + 8 (both = fr mod 8): per instruction the 8 rows of a warp hit
      // 8 different chunks, so the 32 lanes cover the 32 banks once.
      // With half a tile staged, columns 0..127 go first; the second pass waits until their stores have read them.
      uint8_t* stg = s_stg + wg * Cfg::STG_BOXES * Cfg::BOX_BYTES + ((cw & 3) * 16 + fr) * 128 + 4 * fc;
#pragma unroll
      for (int pass = 0; pass < Cfg::PASSES; pass++) {
        ptx::mbar_wait(&stg_ready[wg], (local * Cfg::PASSES + pass) & 1);
#pragma unroll
        for (int jj = 0; jj < Cfg::STG_BOXES * 8; jj++) {
          const int j = pass * Cfg::STG_BOXES * 8 + jj;   // 8-column group of the tile
          const float2 bb = *reinterpret_cast<const float2*>(bias_t + 8 * j + 2 * fc);
#pragma unroll
          for (int h = 0; h < 2; h++) {
            uint32_t* p = reinterpret_cast<uint32_t*>(stg + (jj >> 3) * Cfg::BOX_BYTES + h * 8 * 128 + (((jj & 7) ^ fr) << 4));
            const float2 r = HAS_RES ? unpack_bf16x2(*p) : make_float2(0.f, 0.f);
            *p = pack_bf16x2(epi_apply(acc[4 * j + 2 * h] + bb.x, SPEC & 3, HAS_RES, r.x),
                             epi_apply(acc[4 * j + 2 * h + 1] + bb.y, SPEC & 3, HAS_RES, r.y));
          }
        }
        ptx::fence_proxy_async();   // the TMA stores (async proxy) read what these generic stores wrote
        ptx::mbar_arrive(&stg_full[wg]);
      }
    } else {
      // ---------------- epilogue: register stores through a per-warp fp32 chunk, 8 chunks of 32 columns -----------
      // after the staging round trip, lane (fr, fc) holds columns 8 fc .. 8 fc + 7 of the chunk for rows fr and fr + 8
      float* stg = reinterpret_cast<float*>(s_stg) + cw * 16 * Cfg::STG_LD;
      const int row0 = m_blk * GEMM_BM + wg * 64 + (cw & 3) * 16 + fr;
      bool ok[2];
      EpiRow er[2];
#pragma unroll
      for (int q = 0; q < 2; q++) {
        ok[q] = row0 + 8 * q < M;
        er[q] = epi_row(ep, ok[q] ? row0 + 8 * q : 0, n0);
      }
      uint4 res[2][2];   // [chunk parity][q]: the next chunk's residual is loaded while this one is stored
      auto load_res = [&](int c, uint4 (&r)[2]) {
#pragma unroll
        for (int q = 0; q < 2; q++) {
          const int col = c * 32 + fc * 8;
          r[q] = (HAS_RES && ok[q] && n0 + col < N) ? *reinterpret_cast<const uint4*>(er[q].res_ptr + col)
                                                     : make_uint4(0u, 0u, 0u, 0u);
        }
      };
      load_res(0, res[0]);
#pragma unroll
      for (int c = 0; c < BN / 32; c++) {
        if (c + 1 < BN / 32) load_res(c + 1, res[(c + 1) & 1]);
        __syncwarp();
#pragma unroll
        for (int jj = 0; jj < 4; jj++) {
          const int j = 4 * c + jj;
          *reinterpret_cast<float2*>(stg + fr * Cfg::STG_LD + 8 * jj + 2 * fc) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(stg + (fr + 8) * Cfg::STG_LD + 8 * jj + 2 * fc) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
        __syncwarp();
#pragma unroll
        for (int q = 0; q < 2; q++) {
          const int col = c * 32 + fc * 8;
          if (ok[q] && n0 + col < N) {
            // odd rows read their two halves in the other order: rows fr and fr + 1 (40 floats apart) then hit
            // disjoint banks within a quarter-warp
            const float* src = stg + (fr + 8 * q) * Cfg::STG_LD + fc * 8;
            const int sw = (fr & 1) * 4;
            const float4 h0 = *reinterpret_cast<const float4*>(src + sw);
            const float4 h1 = *reinterpret_cast<const float4*>(src + (4 - sw));
            const float4 u = sw ? h1 : h0, v = sw ? h0 : h1;
            const uint32_t r8[8] = {__float_as_uint(u.x), __float_as_uint(u.y), __float_as_uint(u.z), __float_as_uint(u.w),
                                    __float_as_uint(v.x), __float_as_uint(v.y), __float_as_uint(v.z), __float_as_uint(v.w)};
            epi_store8<SPEC>(er[q], r8, bias_t, col, res[c & 1][q]);
          }
        }
      }
    }
  }
}

// host side (gemm.cu)
int make_tmap_2d(CUtensorMap* out, const void* ptr, int dtype_bf16, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                 uint32_t box_rows, uint32_t box_cols);
int make_tmap_3d(CUtensorMap* out, const void* ptr, int dtype_bf16, uint64_t planes, uint64_t rows, uint64_t cols,
                 uint64_t ld_row, uint64_t ld_plane, uint32_t box_rows, uint32_t box_cols);
// [B, H, W, C] bf16 NHWC activations (C a multiple of 8) seen through an im2col map for the 3x3 pad-1 convolution:
// boxes of 128 pixels x 64 channels, 128B swizzle (the layout of a 128 x 64 tiled A box), zero fill outside.
int make_tmap_im2col_3x3(CUtensorMap* out, const void* ptr, int B, int H, int W, int C);
// tmB must have boxes of bn rows x 64 columns (128 rows for bn = 256).  The epilogue flavour (activation | residual
// << 2) is a template argument of the kernel: ep.act outside 0..3 is B200_ERR_INVALID (the public entries take 0..2).  bn = 256 (the persistent
// kernel) stores by TMA from 8 tiles per CTA up (or with force_tma_epilogue), else from registers.
int gemm_bf16_launch(const CUtensorMap& tmA, const CUtensorMap& tmB, int bn, int M, int N, int K,
                     const GemmEpilogue& ep, cudaStream_t st, bool force_tma_epilogue = false);
// Pick the column-block width for a GEMM with N output columns: 256 (persistent kernel) for large grids, else 128,
// or 64 / 32 when the grid would be under-filled.
int gemm_pick_bn(int M, int N, int sms);
// The implicit 3x3 convolution: tmA from make_tmap_im2col_3x3 over [>= B, H, W, C], tmB over W [N, 9 * cb * 64] with
// boxes of bn rows x 64 columns (bn 32, 64 or 128), M = B * H * W.
int conv3x3_launch(const CUtensorMap& tmA, const CUtensorMap& tmB, int bn, int M, int N, const ConvGeom& cg,
                   const GemmEpilogue& ep, cudaStream_t st);
// Column-block width of the convolution: 128, or 64 / 32 when the grid would be under-filled.
int conv_pick_bn(int M, int N, int sms);

}  // namespace b200
