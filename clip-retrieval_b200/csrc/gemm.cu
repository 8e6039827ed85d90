// Host side of the wgmma GEMM: tensor-map construction, launch, and the stand-alone C-ABI entry.
#include "gemm.cuh"
#include <mutex>
#include <cstdlib>
#include <algorithm>

namespace b200 {

typedef CUresult (*encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static encode_tiled_fn get_encode() {
  static encode_tiled_fn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (encode_tiled_fn)p;
  });
  return fn;
}

// 2-D row-major tensor [rows, cols] with leading dimension ld_elems (16-bit elements), tiled in
// boxes of box_rows x box_cols (box_cols * 2 bytes must be 128: the swizzle span).
int make_tmap_2d(CUtensorMap* out, const void* ptr, int dtype_bf16, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                 uint32_t box_rows, uint32_t box_cols) {
  encode_tiled_fn enc = get_encode();
  B200_CHECK(enc != nullptr, B200_ERR_CUDA, "cuTensorMapEncodeTiled is not available from this driver");
  B200_CHECK(((uintptr_t)ptr & 15) == 0 && (ld_elems * 2) % 16 == 0, B200_ERR_INVALID,
             "tensor map: base and row pitch must be 16-byte aligned (ptr=%p ld=%llu)", ptr,
             (unsigned long long)ld_elems);
  B200_CHECK(box_cols * 2 == 128 && box_rows >= 1 && box_rows <= 256, B200_ERR_INVALID, "tensor map: bad box");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld_elems * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, dtype_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                   const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  B200_CHECK(r == CUDA_SUCCESS, B200_ERR_CUDA, "cuTensorMapEncodeTiled failed with %d", (int)r);
  return B200_OK;
}

// 3-D row-major tensor [planes, rows, cols] (16-bit elements) with row pitch ld_row and plane pitch ld_plane (in
// elements), tiled in boxes of box_rows x box_cols x 1 plane (box_cols * 2 bytes must be 128: the swizzle span).  A box
// that runs past `rows` is clipped at the end of its plane: those rows are read as zeros, never from the next plane.
int make_tmap_3d(CUtensorMap* out, const void* ptr, int dtype_bf16, uint64_t planes, uint64_t rows, uint64_t cols,
                 uint64_t ld_row, uint64_t ld_plane, uint32_t box_rows, uint32_t box_cols) {
  encode_tiled_fn enc = get_encode();
  B200_CHECK(enc != nullptr, B200_ERR_CUDA, "cuTensorMapEncodeTiled is not available from this driver");
  B200_CHECK(((uintptr_t)ptr & 15) == 0 && (ld_row * 2) % 16 == 0 && (ld_plane * 2) % 16 == 0, B200_ERR_INVALID,
             "tensor map: base and pitches must be 16-byte aligned (ptr=%p ld_row=%llu ld_plane=%llu)", ptr,
             (unsigned long long)ld_row, (unsigned long long)ld_plane);
  B200_CHECK(box_cols * 2 == 128 && box_rows >= 1 && box_rows <= 256, B200_ERR_INVALID, "tensor map: bad box");
  cuuint64_t dims[3] = {cols, rows, planes};
  cuuint64_t strides[2] = {ld_row * 2, ld_plane * 2};
  cuuint32_t box[3] = {box_cols, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(out, dtype_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3,
                   const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  B200_CHECK(r == CUDA_SUCCESS, B200_ERR_CUDA, "cuTensorMapEncodeTiled failed with %d", (int)r);
  return B200_OK;
}

// 256-wide persistent tiles once the grid has at least one of them per SM.  Measured on an H100 SXM (700 W,
// tools/gemm_bench.py): at every measured shape from the ViT-H/14 text tower at batch 64 up (156 tiles and more) the
// 256-wide kernel is faster than the 128-wide one, from 1.28x (c_proj of ViT-L/14 image and of ViT-H/14 text at batch
// 64) to 1.8x (ViT-L/14 patch embedding, ViT-H/14 text qkv at batch 64); below one tile per SM (batch 8: 20 .. 80 tiles) the 128-, 64- and 32-wide tiles spread the weight read
// over more SMs and are mostly as fast or faster.
constexpr long GEMM_WIDE_MIN_TILES_PER_SM = 1;

int gemm_pick_bn(int M, int N, int sms) {
  const long mb = (M + GEMM_BM - 1) / GEMM_BM;
  if (mb * ((N + GEMM_WIDE_BN - 1) / GEMM_WIDE_BN) >= GEMM_WIDE_MIN_TILES_PER_SM * sms) return GEMM_WIDE_BN;
  const long tiles128 = mb * ((N + 127) / 128);
  if (tiles128 < sms && N >= 64) {
    const long tiles64 = mb * ((N + 63) / 64);
    return tiles64 < sms ? 32 : 64;
  }
  return 128;
}

template <int BN, int SPEC>
static int launch_bn_spec(const CUtensorMap& tmA, const CUtensorMap& tmB, int M, int N, int K, const GemmEpilogue& ep,
                          cudaStream_t st) {
  using Cfg = GemmCfg<BN>;
  static std::atomic<unsigned long long> configured{0};  // bit per device: the attribute is per context
  auto kern = gemm_bf16_wgmma_kernel<BN, SPEC>;
  int dev = 0;
  B200_CUDA(cudaGetDevice(&dev));
  if (!(configured.load() >> (dev & 63) & 1ull)) {
    B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    configured.fetch_or(1ull << (dev & 63));
  }
  const long tiles = (long)((M + GEMM_BM - 1) / GEMM_BM) * ((N + BN - 1) / BN);
  kern<<<(unsigned)tiles, GEMM_THREADS, Cfg::SMEM_BYTES, st>>>(tmA, tmB, M, N, K, ep);
  B200_LAUNCH_OK();
  return B200_OK;
}

// the epilogue flavour (activation | residual << 2) fixed at compile time; gemm_bf16_launch has checked ep.act (0..3)
template <int BN>
static int launch_bn(const CUtensorMap& tmA, const CUtensorMap& tmB, int M, int N, int K, const GemmEpilogue& ep,
                     cudaStream_t st) {
  switch (ep.act | (ep.residual ? 4 : 0)) {
    case 0: return launch_bn_spec<BN, 0>(tmA, tmB, M, N, K, ep, st);
    case 1: return launch_bn_spec<BN, 1>(tmA, tmB, M, N, K, ep, st);
    case 2: return launch_bn_spec<BN, 2>(tmA, tmB, M, N, K, ep, st);
    case 3: return launch_bn_spec<BN, 3>(tmA, tmB, M, N, K, ep, st);
    case 4: return launch_bn_spec<BN, 4>(tmA, tmB, M, N, K, ep, st);
    case 5: return launch_bn_spec<BN, 5>(tmA, tmB, M, N, K, ep, st);
    case 6: return launch_bn_spec<BN, 6>(tmA, tmB, M, N, K, ep, st);
    default: return launch_bn_spec<BN, 7>(tmA, tmB, M, N, K, ep, st);
  }
}

template <int SPEC, class Cfg>
static int launch_wide_cfg(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC,
                           const CUtensorMap& tmR, int M, int N, int K, const GemmEpilogue& ep, cudaStream_t st) {
  static std::atomic<int> grid_of[64];   // per device: co-resident CTAs (0 until the attributes are set)
  auto kern = gemm_bf16_wgmma_persistent_kernel<SPEC, Cfg>;
  int dev = 0;
  B200_CUDA(cudaGetDevice(&dev));
  int grid = grid_of[dev & 63].load();
  if (grid == 0) {
    B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    int per_sm = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, GEMM_WIDE_THREADS, Cfg::SMEM_BYTES));
    B200_CHECK(per_sm >= 1, B200_ERR_CUDA, "gemm: the persistent kernel does not fit on an SM");
    grid = per_sm * sm_count(dev);
    grid_of[dev & 63].store(grid);
  }
  const long tiles = (long)((M + GEMM_BM - 1) / GEMM_BM) * ((N + GEMM_WIDE_BN - 1) / GEMM_WIDE_BN);
  kern<<<(unsigned)std::min<long>(tiles, grid), GEMM_WIDE_THREADS, Cfg::SMEM_BYTES, st>>>(tmA, tmB, tmC, tmR, M, N, K,
                                                                                        ep);
  B200_LAUNCH_OK();
  return B200_OK;
}

// The TMA-store epilogue (3-stage ring) where every CTA has at least this many tiles; fewer tiles, and the row maps,
// take the register-store epilogue (4-stage ring).  Measured on an H100 SXM (700 W): the TMA stores won at every
// ViT-L/14 batch-1024 layer GEMM (14 tiles per CTA and more), but at the ViT-H/14 text tower at batch 64 (1.2 - 4.7 tiles
// per CTA) `bench.py --workload e2e` was about 2 % slower with them (DESIGN.md §8).
constexpr long GEMM_WIDE_TMA_MIN_TILES_PER_CTA = 8;

// The TMA-store epilogue takes output (and residual) tensor maps of [M, N] with their own leading dimensions, so the
// stores are clipped at M and N; one encode per map per launch.  force_tma: whatever the grid (tests).
template <int SPEC>
static int launch_wide_spec(const CUtensorMap& tmA, const CUtensorMap& tmB, int M, int N, int K, const GemmEpilogue& ep,
                            cudaStream_t st, bool force_tma) {
  CUtensorMap tmC{}, tmR{};
  int dev = 0;
  B200_CUDA(cudaGetDevice(&dev));
  const long tiles = (long)((M + GEMM_BM - 1) / GEMM_BM) * ((N + GEMM_WIDE_BN - 1) / GEMM_WIDE_BN);
  const bool row_map = ep.out_group > 0 || ep.res_row_mod > 0;
  if (row_map || (!force_tma && tiles < GEMM_WIDE_TMA_MIN_TILES_PER_CTA * sm_count(dev)))
    return launch_wide_cfg<SPEC, GemmWideRegCfg>(tmA, tmB, tmC, tmR, M, N, K, ep, st);
  B200_TRY(make_tmap_2d(&tmC, ep.out, 1, (uint64_t)M, (uint64_t)N, (uint64_t)ep.out_ld, GEMM_WIDE_BOX, GEMM_WIDE_BOX));
  if (ep.residual != nullptr)
    B200_TRY(make_tmap_2d(&tmR, ep.residual, 1, (uint64_t)M, (uint64_t)N, (uint64_t)ep.res_ld, GEMM_WIDE_BOX,
                          GEMM_WIDE_BOX));
  return launch_wide_cfg<SPEC, GemmWideTmaCfg>(tmA, tmB, tmC, tmR, M, N, K, ep, st);
}

static int launch_wide(const CUtensorMap& tmA, const CUtensorMap& tmB, int M, int N, int K, const GemmEpilogue& ep,
                       cudaStream_t st, bool force_tma) {
  switch (ep.act | (ep.residual ? 4 : 0)) {
    case 0: return launch_wide_spec<0>(tmA, tmB, M, N, K, ep, st, force_tma);
    case 1: return launch_wide_spec<1>(tmA, tmB, M, N, K, ep, st, force_tma);
    case 2: return launch_wide_spec<2>(tmA, tmB, M, N, K, ep, st, force_tma);
    case 3: return launch_wide_spec<3>(tmA, tmB, M, N, K, ep, st, force_tma);
    case 4: return launch_wide_spec<4>(tmA, tmB, M, N, K, ep, st, force_tma);
    case 5: return launch_wide_spec<5>(tmA, tmB, M, N, K, ep, st, force_tma);
    case 6: return launch_wide_spec<6>(tmA, tmB, M, N, K, ep, st, force_tma);
    default: return launch_wide_spec<7>(tmA, tmB, M, N, K, ep, st, force_tma);
  }
}

int gemm_bf16_launch(const CUtensorMap& tmA, const CUtensorMap& tmB, int bn, int M, int N, int K,
                     const GemmEpilogue& ep, cudaStream_t st, bool force_tma_epilogue) {
  B200_CHECK(M >= 1 && N >= 8 && K >= 8 && N % 8 == 0 && K % 8 == 0, B200_ERR_INVALID,
             "gemm: need M>=1 and N, K multiples of 8 (M=%d N=%d K=%d)", M, N, K);
  B200_CHECK(ep.out != nullptr && ep.out_ld % 8 == 0 && ((uintptr_t)ep.out & 15) == 0, B200_ERR_INVALID,
             "gemm: output must be 16-byte aligned with ld %% 8 == 0");
  B200_CHECK(ep.residual == nullptr || (ep.res_ld % 8 == 0 && ((uintptr_t)ep.residual & 15) == 0), B200_ERR_INVALID,
             "gemm: residual must be 16-byte aligned with ld %% 8 == 0");
  B200_CHECK(ep.act >= 0 && ep.act <= ACT_RELU, B200_ERR_INVALID, "gemm: act=%d", ep.act);
  if (bn == GEMM_WIDE_BN) return launch_wide(tmA, tmB, M, N, K, ep, st, force_tma_epilogue);
  if (bn == 128) return launch_bn<128>(tmA, tmB, M, N, K, ep, st);
  if (bn == 64) return launch_bn<64>(tmA, tmB, M, N, K, ep, st);
  if (bn == 32) return launch_bn<32>(tmA, tmB, M, N, K, ep, st);
  set_error("gemm: unsupported column block %d", bn);
  return B200_ERR_INVALID;
}

}  // namespace b200

using namespace b200;

// The stand-alone entries: A [M, K] and W [N, K] contiguous, everything else as the epilogue says.  bn = 0 takes
// gemm_pick_bn's width.
// The public entries take activations 0..2: ACT_RELU is internal to the ResNet tower and its convolution entry.
static int gemm_entry(const void* d_A, const void* d_W, int M, int N, int K, const GemmEpilogue& ep, int bn, int device,
                      void* stream, bool force_tma_epilogue = false) {
  B200_CHECK(d_A && d_W && ep.out, B200_ERR_INVALID, "gemm: null operand");
  B200_CHECK(ep.act >= 0 && ep.act <= 2, B200_ERR_INVALID, "gemm: act=%d", ep.act);
  B200_CHECK(bn == 0 || bn == 32 || bn == 64 || bn == 128 || bn == GEMM_WIDE_BN, B200_ERR_INVALID, "gemm: unsupported column block %d", bn);
  DeviceGuard g(device);
  if (bn == 0) bn = gemm_pick_bn(M, N, sm_count(device));
  CUtensorMap tmA, tmB;
  B200_TRY(make_tmap_2d(&tmA, d_A, 1, (uint64_t)M, (uint64_t)K, (uint64_t)K, GEMM_BM, GEMM_BK));
  B200_TRY(make_tmap_2d(&tmB, d_W, 1, (uint64_t)N, (uint64_t)K, (uint64_t)K, (uint32_t)std::min(bn, 128), GEMM_BK));
  return gemm_bf16_launch(tmA, tmB, bn, M, N, K, ep, (cudaStream_t)stream, force_tma_epilogue);
}

extern "C" int b200_gemm_bf16_device(const void* d_A, const void* d_W, const float* d_bias, const void* d_residual,
                                     void* d_C, int M, int N, int K, int act, int device, void* stream) {
  GemmEpilogue ep;
  ep.bias = d_bias;
  ep.residual = (const __nv_bfloat16*)d_residual;
  ep.res_ld = N;
  ep.out = (__nv_bfloat16*)d_C;
  ep.out_ld = N;
  ep.act = act;
  return gemm_entry(d_A, d_W, M, N, K, ep, 0, device, stream);
}

extern "C" int b200_gemm_bf16_ex_device(const void* d_A, const void* d_W, void* d_C, int M, int N, int K,
                                        const b200_gemm_epilogue* e, int bn, int flags, int device, void* stream) {
  B200_CHECK(e != nullptr, B200_ERR_INVALID, "gemm: null epilogue");
  // bit 1: the persistent kernel's TMA-store epilogue whatever the grid size (the tests reach it at small shapes)
  B200_CHECK((flags & ~2) == 0, B200_ERR_INVALID, "gemm: flags=%d (only bit 1 is defined)", flags);
  B200_CHECK(!e->reserved0 && !e->reserved1 && e->reserved2 == 0 && !e->reserved3, B200_ERR_INVALID,
             "gemm: the reserved members of b200_gemm_epilogue must be zero (the LayerNorm fold was removed)");
  GemmEpilogue ep;
  ep.bias = e->bias;
  ep.residual = (const __nv_bfloat16*)e->residual;
  ep.res_ld = e->res_ld > 0 ? e->res_ld : N;
  ep.res_row_mod = e->res_row_mod;
  ep.res_row_off = e->res_row_off;
  ep.out = (__nv_bfloat16*)d_C;
  ep.out_ld = e->out_ld > 0 ? e->out_ld : N;
  ep.out_group = e->out_group;
  ep.act = e->act;
  return gemm_entry(d_A, d_W, M, N, K, ep, bn, device, stream, (flags & 2) != 0);
}
