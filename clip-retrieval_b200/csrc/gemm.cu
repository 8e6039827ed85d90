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

int gemm_pick_bn(int M, int N, int sms) {
  const long mb = (M + GEMM_BM - 1) / GEMM_BM;
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

// the epilogue flavour (activation | residual << 2) fixed at compile time unless the LayerNorm fold or the row
// statistics are in use
template <int BN>
static int launch_bn(const CUtensorMap& tmA, const CUtensorMap& tmB, int M, int N, int K, const GemmEpilogue& ep,
                     cudaStream_t st) {
  const bool plain = ep.ln_stats == nullptr && ep.stats_out == nullptr && ep.ln_c == nullptr &&
                     ep.act >= 0 && ep.act <= 2;
  if (plain) {
    switch ((ep.act & 3) | (ep.residual ? 4 : 0)) {
      case 0: return launch_bn_spec<BN, 0>(tmA, tmB, M, N, K, ep, st);
      case 1: return launch_bn_spec<BN, 1>(tmA, tmB, M, N, K, ep, st);
      case 2: return launch_bn_spec<BN, 2>(tmA, tmB, M, N, K, ep, st);
      case 4: return launch_bn_spec<BN, 4>(tmA, tmB, M, N, K, ep, st);
      case 5: return launch_bn_spec<BN, 5>(tmA, tmB, M, N, K, ep, st);
      case 6: return launch_bn_spec<BN, 6>(tmA, tmB, M, N, K, ep, st);
      default: break;
    }
  }
  return launch_bn_spec<BN, -1>(tmA, tmB, M, N, K, ep, st);
}

int gemm_bf16_launch(const CUtensorMap& tmA, const CUtensorMap& tmB, int bn, int M, int N, int K,
                     const GemmEpilogue& ep, cudaStream_t st) {
  B200_CHECK(M >= 1 && N >= 8 && K >= 8 && N % 8 == 0 && K % 8 == 0, B200_ERR_INVALID,
             "gemm: need M>=1 and N, K multiples of 8 (M=%d N=%d K=%d)", M, N, K);
  B200_CHECK(ep.out != nullptr && ep.out_ld % 8 == 0 && ((uintptr_t)ep.out & 15) == 0, B200_ERR_INVALID,
             "gemm: output must be 16-byte aligned with ld %% 8 == 0");
  B200_CHECK(ep.residual == nullptr || (ep.res_ld % 8 == 0 && ((uintptr_t)ep.residual & 15) == 0), B200_ERR_INVALID,
             "gemm: residual must be 16-byte aligned with ld %% 8 == 0");
  B200_CHECK(ep.stats_out == nullptr || (N % 64 == 0 && bn >= 128), B200_ERR_INVALID,
             "gemm: row statistics need N %% 64 == 0 and tiles of at least 128 columns (N=%d, bn=%d)", N, bn);
  B200_CHECK(ep.ln_stats == nullptr || (ep.ln_c != nullptr && ep.ln_w > 0 && ep.ln_w % 64 == 0), B200_ERR_INVALID,
             "gemm: folded LayerNorm needs c and a row width that is a multiple of 64 (ln_w=%d)", ep.ln_w);
  B200_CHECK(ep.ln_stats == nullptr || ep.ln_w <= 64 * LN_MAX_SLOTS, B200_ERR_UNSUPPORTED, "gemm: folded LayerNorm supports rows of at most %d columns", 64 * LN_MAX_SLOTS);
  if (bn == 128) return launch_bn<128>(tmA, tmB, M, N, K, ep, st);
  if (bn == 64) return launch_bn<64>(tmA, tmB, M, N, K, ep, st);
  if (bn == 32) return launch_bn<32>(tmA, tmB, M, N, K, ep, st);
  set_error("gemm: unsupported column block %d", bn);
  return B200_ERR_INVALID;
}

}  // namespace b200

using namespace b200;

extern "C" int b200_gemm_bf16_device(const void* d_A, const void* d_W, const float* d_bias, const void* d_residual,
                                     void* d_C, int M, int N, int K, int act, int device, void* stream) {
  B200_CHECK(d_A && d_W && d_C, B200_ERR_INVALID, "gemm: null operand");
  B200_CHECK(act >= 0 && act <= 2, B200_ERR_INVALID, "gemm: act=%d", act);
  DeviceGuard g(device);
  const int sms = sm_count(device);
  const int bn = gemm_pick_bn(M, N, sms);
  CUtensorMap tmA, tmB;
  B200_TRY(make_tmap_2d(&tmA, d_A, 1, (uint64_t)M, (uint64_t)K, (uint64_t)K, GEMM_BM, GEMM_BK));
  B200_TRY(make_tmap_2d(&tmB, d_W, 1, (uint64_t)N, (uint64_t)K, (uint64_t)K, (uint32_t)bn, GEMM_BK));
  GemmEpilogue ep;
  ep.bias = d_bias;
  ep.residual = (const __nv_bfloat16*)d_residual;
  ep.res_ld = N;
  ep.out = (__nv_bfloat16*)d_C;
  ep.out_ld = N;
  ep.act = act;
  return gemm_bf16_launch(tmA, tmB, bn, M, N, K, ep, (cudaStream_t)stream);
}
