// Convolutions and the small kernels of the ResNet image tower (OpenAI's ModifiedResNet, resnet.cu):
//   - the 3x3 stride-1 pad-1 convolution as an implicit GEMM on the 128-row wgmma kernel (gemm.cuh
//     conv3x3_bf16_wgmma_kernel): activations stay NHWC bf16 [B*H*W, C]; the producer reads each 128 x 64 A box with
//     one im2col TMA load at the tap's offset, so no im2col buffer exists.  The weight is packed [N, 9 * C64] (C64 =
//     ceil(C / 64) * 64, K index = (3 r + s) * C64 + c, zero columns in the padding); borders and channels >= C come
//     from TMA's zero fill.  Roofline: tensor pipe, 2 * M * N * 9 * C64 flops (the padding included); the A traffic is
//     9 * C64 / C times the activation, mostly from L2.
//   - the stem gather: the 27 taps of the stride-2 stem convolution into a [B * (S/2)^2, 64] patch matrix;
//   - AvgPool2d(k) on NHWC bf16, accumulated in fp32;
//   - the attention-pool tokens: spatial mean as token 0, + positional embedding.
#include "common.cuh"
#include "embed_kernels.cuh"
#include "gemm.cuh"
#include <algorithm>
#include <atomic>
#include <mutex>

namespace b200 {

typedef CUresult (*encode_im2col_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*,
                                     CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                     CUtensorMapFloatOOBfill);

static encode_im2col_fn get_encode_im2col() {
  static encode_im2col_fn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (encode_im2col_fn)p;
  });
  return fn;
}

// The bounding box of the base pixel runs from -1 (lower corner) to dim - 2 (upper corner -1): the H x W output
// pixels of a 3x3 pad-1 convolution, whose tap (r, s) reads input pixel (h - 1 + r, w - 1 + s).
int make_tmap_im2col_3x3(CUtensorMap* out, const void* ptr, int B, int H, int W, int C) {
  encode_im2col_fn enc = get_encode_im2col();
  B200_CHECK(enc != nullptr, B200_ERR_CUDA, "cuTensorMapEncodeIm2col is not available from this driver");
  B200_CHECK(((uintptr_t)ptr & 15) == 0 && C % 8 == 0 && B >= 1 && H >= 1 && W >= 1, B200_ERR_INVALID,
             "im2col map: base 16-byte aligned and C a multiple of 8 (ptr=%p C=%d)", ptr, C);
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  int lower[2] = {-1, -1}, upper[2] = {-1, -1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, lower, upper,
                   GEMM_BK, GEMM_BM, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  B200_CHECK(r == CUDA_SUCCESS, B200_ERR_CUDA, "cuTensorMapEncodeIm2col failed with %d", (int)r);
  return B200_OK;
}

int conv_pick_bn(int M, int N, int sms) {
  const long mb = (M + GEMM_BM - 1) / GEMM_BM;
  if (mb * ((N + 127) / 128) < sms && N >= 64) return mb * ((N + 63) / 64) < sms ? 32 : 64;
  return 128;
}

template <int BN, int SPEC>
static int conv_launch_spec(const CUtensorMap& tmA, const CUtensorMap& tmB, int M, int N, const ConvGeom& cg,
                            const GemmEpilogue& ep, cudaStream_t st) {
  using Cfg = GemmCfg<BN>;
  static std::atomic<unsigned long long> configured{0};  // bit per device: the attribute is per context
  auto kern = conv3x3_bf16_wgmma_kernel<BN, SPEC>;
  int dev = 0;
  B200_CUDA(cudaGetDevice(&dev));
  if (!(configured.load() >> (dev & 63) & 1ull)) {
    B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    configured.fetch_or(1ull << (dev & 63));
  }
  const long tiles = (long)((M + GEMM_BM - 1) / GEMM_BM) * ((N + BN - 1) / BN);
  kern<<<(unsigned)tiles, GEMM_THREADS, Cfg::SMEM_BYTES, st>>>(tmA, tmB, M, N, 9 * cg.cb * GEMM_BK, ep, cg);
  B200_LAUNCH_OK();
  return B200_OK;
}

template <int BN>
static int conv_launch_bn(const CUtensorMap& tmA, const CUtensorMap& tmB, int M, int N, const ConvGeom& cg,
                          const GemmEpilogue& ep, cudaStream_t st) {
  switch (ep.act | (ep.residual ? 4 : 0)) {
    case 0: return conv_launch_spec<BN, 0>(tmA, tmB, M, N, cg, ep, st);
    case 3: return conv_launch_spec<BN, 3>(tmA, tmB, M, N, cg, ep, st);
    case 4: return conv_launch_spec<BN, 4>(tmA, tmB, M, N, cg, ep, st);
    default: return conv_launch_spec<BN, 7>(tmA, tmB, M, N, cg, ep, st);
  }
}

int conv3x3_launch(const CUtensorMap& tmA, const CUtensorMap& tmB, int bn, int M, int N, const ConvGeom& cg,
                   const GemmEpilogue& ep, cudaStream_t st) {
  B200_CHECK(M >= 1 && N >= 8 && N % 8 == 0 && cg.cb >= 1 && cg.H >= 1 && cg.W >= 1, B200_ERR_INVALID,
             "conv3x3: need M>=1, N a multiple of 8 (M=%d N=%d)", M, N);
  B200_CHECK(ep.out != nullptr && ep.out_ld % 8 == 0 && ((uintptr_t)ep.out & 15) == 0, B200_ERR_INVALID,
             "conv3x3: output must be 16-byte aligned with ld %% 8 == 0");
  B200_CHECK(ep.residual == nullptr || (ep.res_ld % 8 == 0 && ((uintptr_t)ep.residual & 15) == 0), B200_ERR_INVALID,
             "conv3x3: residual must be 16-byte aligned with ld %% 8 == 0");
  B200_CHECK(ep.act == ACT_NONE || ep.act == ACT_RELU, B200_ERR_INVALID, "conv3x3: act=%d (none or relu)", ep.act);
  B200_CHECK(ep.out_group == 0 && ep.res_row_mod == 0, B200_ERR_INVALID, "conv3x3: no row maps");
  if (bn == 128) return conv_launch_bn<128>(tmA, tmB, M, N, cg, ep, st);
  if (bn == 64) return conv_launch_bn<64>(tmA, tmB, M, N, cg, ep, st);
  if (bn == 32) return conv_launch_bn<32>(tmA, tmB, M, N, cg, ep, st);
  set_error("conv3x3: unsupported column block %d", bn);
  return B200_ERR_INVALID;
}

// cols[b * g * g + oy * g + ox, c * 9 + r * 3 + s] = px[b, c, 2 oy - 1 + r, 2 ox - 1 + s] (0 outside), g = S / 2
__global__ void stem_gather_kernel(const float* __restrict__ px, __nv_bfloat16* __restrict__ cols, int S, int g, int Kp,
                                   long total) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int k = (int)(i % 27);
  const long row = i / 27;
  const int ox = (int)(row % g), oy = (int)((row / g) % g);
  const long b = row / ((long)g * g);
  const int c = k / 9, r = (k / 3) % 3, s = k % 3;
  const int y = 2 * oy - 1 + r, x = 2 * ox - 1 + s;
  const float v = (y >= 0 && y < S && x >= 0 && x < S) ? px[((b * 3 + c) * S + y) * S + x] : 0.0f;
  cols[row * Kp + k] = __float2bfloat16_rn(v);
}

int stem_gather(const float* px, __nv_bfloat16* cols, int B, int S, int Kp, cudaStream_t st) {
  if (B == 0) return B200_OK;
  const int g = S / 2;
  const long total = (long)B * g * g * 27;
  stem_gather_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(px, cols, S, g, Kp, total);
  B200_LAUNCH_OK();
  return B200_OK;
}

// 8 channels per thread: out[b, oy, ox, c..c+7] = (sum over the k x k window, row-major, in fp32) / k^2
__global__ void avgpool_kernel(const __nv_bfloat16* __restrict__ in, __nv_bfloat16* __restrict__ out, int H, int W,
                               int C, int k, int Ho, int Wo, long total) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c8 = C / 8;
  const int c = (int)(i % c8) * 8;
  const long p = i / c8;
  const int ox = (int)(p % Wo), oy = (int)((p / Wo) % Ho);
  const long b = p / ((long)Wo * Ho);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int dy = 0; dy < k; dy++)
    for (int dx = 0; dx < k; dx++) {
      const uint4 u = *reinterpret_cast<const uint4*>(in + ((b * H + oy * k + dy) * W + ox * k + dx) * C + c);
      const uint32_t q[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const float2 f = unpack_bf16x2(q[j]);
        acc[2 * j] += f.x;
        acc[2 * j + 1] += f.y;
      }
    }
  const float inv = 1.0f / (float)(k * k);
  uint4 o;
  o.x = pack_bf16x2(acc[0] * inv, acc[1] * inv);
  o.y = pack_bf16x2(acc[2] * inv, acc[3] * inv);
  o.z = pack_bf16x2(acc[4] * inv, acc[5] * inv);
  o.w = pack_bf16x2(acc[6] * inv, acc[7] * inv);
  *reinterpret_cast<uint4*>(out + p * C + c) = o;
}

int avgpool_nhwc(const __nv_bfloat16* in, __nv_bfloat16* out, int B, int H, int W, int C, int k, cudaStream_t st) {
  B200_CHECK(k >= 1 && C % 8 == 0 && H >= k && W >= k, B200_ERR_INVALID, "avgpool: k=%d C=%d H=%d W=%d", k, C, H, W);
  if (B == 0) return B200_OK;
  const int Ho = H / k, Wo = W / k;
  const long total = (long)B * Ho * Wo * (C / 8);
  avgpool_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(in, out, H, W, C, k, Ho, Wo, total);
  B200_LAUNCH_OK();
  return B200_OK;
}

// out[b * T + 0, c] = bf16(mean over hw of x[b * HW + hw, c] + pos[0, c]); out[b * T + t, c] = bf16(x[b * HW + t - 1, c]
// + pos[t, c]) for t >= 1 (T = HW + 1).  The mean is an fp32 sum in hw order divided by HW.
__global__ void __launch_bounds__(256)
attnpool_tokens_kernel(const __nv_bfloat16* __restrict__ x, int HW, int C, const float* __restrict__ pos,
                       __nv_bfloat16* __restrict__ out) {
  const int t = blockIdx.x, b = blockIdx.y, T = HW + 1;
  const __nv_bfloat16* xb = x + (size_t)b * HW * C;
  __nv_bfloat16* o = out + ((size_t)b * T + t) * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float v;
    if (t == 0) {
      float s = 0.f;
      for (int hw = 0; hw < HW; hw++) s += __bfloat162float(xb[(size_t)hw * C + c]);
      v = s / (float)HW;
    } else {
      v = __bfloat162float(xb[(size_t)(t - 1) * C + c]);
    }
    o[c] = __float2bfloat16_rn(v + pos[(size_t)t * C + c]);
  }
}

int attnpool_tokens(const __nv_bfloat16* x, int B, int HW, int C, const float* pos, __nv_bfloat16* out,
                    cudaStream_t st) {
  if (B == 0) return B200_OK;
  attnpool_tokens_kernel<<<dim3(HW + 1, B), 256, 0, st>>>(x, HW, C, pos, out);
  B200_LAUNCH_OK();
  return B200_OK;
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_conv_bf16_device(const void* d_x, int B, int H, int W, int C, const void* d_w, int N, int ksize, void* d_out,
                          const b200_gemm_epilogue* e, int bn, int device, void* stream) {
  B200_CHECK(d_x && d_w && d_out && e && B >= 1 && H >= 1 && W >= 1 && C >= 8 && C % 8 == 0 && (ksize == 1 || ksize == 3),
             B200_ERR_INVALID, "conv: bad argument");
  B200_CHECK(!e->reserved0 && !e->reserved1 && e->reserved2 == 0 && !e->reserved3 && e->out_group == 0 &&
                 e->res_row_mod == 0 && e->act >= 0 && e->act <= ACT_RELU,
             B200_ERR_INVALID, "conv: epilogue (act 0..3, no row maps, reserved members zero)");
  const long M = (long)B * H * W;
  B200_CHECK(M < (1l << 31), B200_ERR_INVALID, "conv: B*H*W too large");
  GemmEpilogue ep;
  ep.bias = e->bias;
  ep.residual = (const __nv_bfloat16*)e->residual;
  ep.res_ld = e->res_ld > 0 ? e->res_ld : N;
  ep.out = (__nv_bfloat16*)d_out;
  ep.out_ld = e->out_ld > 0 ? e->out_ld : N;
  ep.act = e->act;
  DeviceGuard g(device);
  CUtensorMap tmA, tmB;
  if (ksize == 1) {
    // the 1x1 convolution is the GEMM of [B*H*W, C] rows; bn 256 is the persistent kernel
    B200_CHECK(bn == 0 || bn == 32 || bn == 64 || bn == 128 || bn == GEMM_WIDE_BN, B200_ERR_INVALID, "conv: bn %d", bn);
    if (bn == 0) bn = gemm_pick_bn((int)M, N, sm_count(device));
    B200_TRY(make_tmap_2d(&tmA, d_x, 1, (uint64_t)M, (uint64_t)C, (uint64_t)C, GEMM_BM, GEMM_BK));
    B200_TRY(make_tmap_2d(&tmB, d_w, 1, (uint64_t)N, (uint64_t)C, (uint64_t)C, (uint32_t)std::min(bn, 128), GEMM_BK));
    return gemm_bf16_launch(tmA, tmB, bn, (int)M, N, C, ep, (cudaStream_t)stream);
  }
  B200_CHECK(bn == 0 || bn == 32 || bn == 64 || bn == 128, B200_ERR_INVALID, "conv3x3: bn %d", bn);
  if (bn == 0) bn = conv_pick_bn((int)M, N, sm_count(device));
  ConvGeom cg;
  cg.H = H; cg.W = W; cg.cb = (C + GEMM_BK - 1) / GEMM_BK;
  const uint64_t K = (uint64_t)9 * cg.cb * GEMM_BK;
  B200_TRY(make_tmap_im2col_3x3(&tmA, d_x, B, H, W, C));
  B200_TRY(make_tmap_2d(&tmB, d_w, 1, (uint64_t)N, K, K, (uint32_t)bn, GEMM_BK));
  return conv3x3_launch(tmA, tmB, bn, (int)M, N, cg, ep, (cudaStream_t)stream);
}

int b200_stem_gather_device(const float* d_pixels, int B, int S, void* d_cols, int device, void* stream) {
  B200_CHECK(B >= 0 && S >= 2 && S % 2 == 0 && (B == 0 || (d_pixels && d_cols)), B200_ERR_INVALID,
             "stem_gather: bad argument");
  DeviceGuard g(device);
  return stem_gather(d_pixels, (__nv_bfloat16*)d_cols, B, S, GEMM_BK, (cudaStream_t)stream);
}

int b200_avgpool_bf16_device(const void* d_in, int B, int H, int W, int C, int k, void* d_out, int device,
                             void* stream) {
  B200_CHECK(B >= 0 && (B == 0 || (d_in && d_out)), B200_ERR_INVALID, "avgpool: bad argument");
  DeviceGuard g(device);
  return avgpool_nhwc((const __nv_bfloat16*)d_in, (__nv_bfloat16*)d_out, B, H, W, C, k, (cudaStream_t)stream);
}

int b200_attnpool_tokens_device(const void* d_x, int B, int HW, int C, const float* d_pos, void* d_out, int device,
                                void* stream) {
  B200_CHECK(B >= 0 && HW >= 1 && C >= 1 && (B == 0 || (d_x && d_pos && d_out)), B200_ERR_INVALID,
             "attnpool_tokens: bad argument");
  DeviceGuard g(device);
  return attnpool_tokens((const __nv_bfloat16*)d_x, B, HW, C, d_pos, (__nv_bfloat16*)d_out, (cudaStream_t)stream);
}

}  // extern "C"
