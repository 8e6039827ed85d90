// The ConvNeXt tower's own kernels (convnext.cu): the depthwise 7x7 convolution fused with the block's LayerNorm, the
// LayerNorm + 2x2 space-to-depth in front of each downsample GEMM, and the head's spatial mean + LayerNorm.  NHWC bf16
// activations, every sum and statistic in fp32 in a fixed order, so each result is deterministic.
#include "embed_kernels.cuh"
#include <algorithm>

namespace b200 {

// ---- dwconv7_ln ------------------------------------------------------------------------------------------------------
// A block owns DW_P consecutive output pixels of one row (b, h, w0 .. w0 + DW_P - 1) and all C channels.  Phase 1: each
// thread takes channel pairs; for each of the 7 input rows it holds the DW_P + 6 input pixels of its pair in registers
// (the horizontal halo is reused there, the vertical one comes from the 7 neighbouring rows' blocks through L2) and
// sums the taps as fma chains in the order r = 0..6, s = 0..6, then adds the bias; the fp32 results go to shared
// memory [DW_P][C].  Phase 2: a warp per pixel takes the mean and then the variance of its row from shared memory and
// writes LN(y) * g + b as bf16 (y itself when g is null).
constexpr int DW_P = 8;

__global__ void __launch_bounds__(256)
dwconv7_ln_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ w49, const float* __restrict__ bias,
                  const float* __restrict__ g, const float* __restrict__ be, float eps, __nv_bfloat16* __restrict__ out,
                  int H, int W, int C) {
  extern __shared__ float s_y[];   // [DW_P][C]
  const int w0 = blockIdx.x * DW_P, h = blockIdx.y, b = blockIdx.z;
  const int pairs = C >> 1;
  for (int cp = threadIdx.x; cp < pairs; cp += blockDim.x) {
    const int c = cp * 2;
    float2 acc[DW_P];
#pragma unroll
    for (int p = 0; p < DW_P; p++) acc[p] = make_float2(0.f, 0.f);
    for (int r = 0; r < 7; r++) {
      const int ih = h + r - 3;
      if (ih < 0 || ih >= H) continue;   // the same for every thread of the block
      const __nv_bfloat16* row = x + ((size_t)b * H + ih) * W * C + c;
      float2 in[DW_P + 6];
#pragma unroll
      for (int k = 0; k < DW_P + 6; k++) {
        const int iw = w0 + k - 3;
        in[k] = (iw >= 0 && iw < W) ? __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(row + (size_t)iw * C))
                                    : make_float2(0.f, 0.f);
      }
#pragma unroll
      for (int s = 0; s < 7; s++) {
        const float2 wv = *reinterpret_cast<const float2*>(w49 + (size_t)(r * 7 + s) * C + c);
#pragma unroll
        for (int p = 0; p < DW_P; p++) {
          acc[p].x = fmaf(wv.x, in[p + s].x, acc[p].x);
          acc[p].y = fmaf(wv.y, in[p + s].y, acc[p].y);
        }
      }
    }
    const float2 bv = *reinterpret_cast<const float2*>(bias + c);
#pragma unroll
    for (int p = 0; p < DW_P; p++) {
      s_y[p * C + c] = acc[p].x + bv.x;
      s_y[p * C + c + 1] = acc[p].y + bv.y;
    }
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const int np = min(DW_P, W - w0);
  for (int p = threadIdx.x >> 5; p < np; p += nwarps) {
    const float* y = s_y + p * C;
    __nv_bfloat162* dst = reinterpret_cast<__nv_bfloat162*>(out + (((size_t)b * H + h) * W + w0 + p) * C);
    if (g == nullptr) {
      for (int cp = lane; cp < pairs; cp += 32) dst[cp] = __floats2bfloat162_rn(y[2 * cp], y[2 * cp + 1]);
      continue;
    }
    float sum = 0.f;
    for (int j = lane; j < C; j += 32) sum += y[j];
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum / (float)C;
    float ss = 0.f;
    for (int j = lane; j < C; j += 32) {
      const float d = y[j] - mean;
      ss += d * d;
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float rstd = rsqrtf(ss / (float)C + eps);
    for (int cp = lane; cp < pairs; cp += 32) {
      const int j = 2 * cp;
      dst[cp] = __floats2bfloat162_rn((y[j] - mean) * rstd * g[j] + be[j], (y[j + 1] - mean) * rstd * g[j + 1] + be[j + 1]);
    }
  }
}

int dwconv7_ln(const __nv_bfloat16* x, const float* w49, const float* bias, const float* gamma, const float* beta,
               float eps, __nv_bfloat16* out, int B, int H, int W, int C, cudaStream_t st) {
  B200_CHECK(C >= 64 && C % 64 == 0 && C <= 3072 && H >= 1 && W >= 1, B200_ERR_UNSUPPORTED,
             "dwconv7_ln: C=%d (need a multiple of 64, <= 3072), H=%d W=%d", C, H, W);
  if (B == 0) return B200_OK;
  const size_t smem = (size_t)DW_P * C * sizeof(float);
  B200_CUDA(cudaFuncSetAttribute(dwconv7_ln_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int threads = std::min(C / 2, 256);
  dwconv7_ln_kernel<<<dim3((W + DW_P - 1) / DW_P, H, B), threads, smem, st>>>(x, w49, bias, gamma, beta, eps, out, H, W,
                                                                               C);
  B200_LAUNCH_OK();
  return B200_OK;
}

// ---- ln_s2d ----------------------------------------------------------------------------------------------------------
// A warp per input pixel (b, ih, iw): its C channels in registers (CPL 16-byte chunks per lane), mean then variance,
// and LN(x) * g + b written at row (b, ih / 2, iw / 2), columns ((ih & 1) * 2 + (iw & 1)) * C + c of the [.., 4C]
// matrix the downsample GEMM reads.
template <int CPL>
__global__ void __launch_bounds__(256)
ln_s2d_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ g, const float* __restrict__ be, float eps,
              __nv_bfloat16* __restrict__ out, int64_t pixels, int H, int W, int C) {
  const int lane = threadIdx.x & 31;
  const int64_t pix = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (pix >= pixels) return;
  const int chunks = C >> 3;
  const __nv_bfloat16* src = x + pix * C;
  float v[CPL][8];
  float sum = 0.f;
#pragma unroll
  for (int c = 0; c < CPL; c++) {
    const int ci = c * 32 + lane;
    const uint4 u = ci < chunks ? *reinterpret_cast<const uint4*>(src + ci * 8) : make_uint4(0u, 0u, 0u, 0u);
    const __nv_bfloat162* hp = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const float2 f = __bfloat1622float2(hp[j]);
      v[c][2 * j] = f.x;
      v[c][2 * j + 1] = f.y;
      sum += f.x + f.y;   // chunks past the row are zeros
    }
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / (float)C;
  float ss = 0.f;
#pragma unroll
  for (int c = 0; c < CPL; c++)
    if (c * 32 + lane < chunks) {
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const float d = v[c][j] - mean;
        ss += d * d;
      }
    }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float rstd = rsqrtf(ss / (float)C + eps);
  const int64_t hw = (int64_t)H * W;
  const int64_t bi = pix / hw;
  const int rem = (int)(pix - bi * hw), ih = rem / W, iw = rem - ih * W;
  const int Ho = H >> 1, Wo = W >> 1;
  __nv_bfloat16* dst = out + ((bi * Ho + (ih >> 1)) * Wo + (iw >> 1)) * 4 * C + (size_t)((ih & 1) * 2 + (iw & 1)) * C;
#pragma unroll
  for (int c = 0; c < CPL; c++) {
    const int ci = c * 32 + lane;
    if (ci < chunks) {
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int k = ci * 8 + 2 * j;
        __nv_bfloat162 t = __floats2bfloat162_rn((v[c][2 * j] - mean) * rstd * g[k] + be[k],
                                                 (v[c][2 * j + 1] - mean) * rstd * g[k + 1] + be[k + 1]);
        o[j] = *reinterpret_cast<uint32_t*>(&t);
      }
      *reinterpret_cast<uint4*>(dst + ci * 8) = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
}

int ln_s2d(const __nv_bfloat16* x, const float* gamma, const float* beta, float eps, __nv_bfloat16* out, int B, int H,
           int W, int C, cudaStream_t st) {
  B200_CHECK(C >= 8 && C % 8 == 0 && C <= 1536 && H % 2 == 0 && W % 2 == 0 && H >= 2 && W >= 2, B200_ERR_UNSUPPORTED,
             "ln_s2d: C=%d (need a multiple of 8, <= 1536), H=%d W=%d even", C, H, W);
  if (B == 0) return B200_OK;
  const int64_t pixels = (int64_t)B * H * W;
  const unsigned grid = (unsigned)((pixels + 7) / 8);
  switch ((C / 8 + 31) / 32) {
    case 1: ln_s2d_kernel<1><<<grid, 256, 0, st>>>(x, gamma, beta, eps, out, pixels, H, W, C); break;
    case 2: ln_s2d_kernel<2><<<grid, 256, 0, st>>>(x, gamma, beta, eps, out, pixels, H, W, C); break;
    case 3: ln_s2d_kernel<3><<<grid, 256, 0, st>>>(x, gamma, beta, eps, out, pixels, H, W, C); break;
    case 4: ln_s2d_kernel<4><<<grid, 256, 0, st>>>(x, gamma, beta, eps, out, pixels, H, W, C); break;
    case 5: ln_s2d_kernel<5><<<grid, 256, 0, st>>>(x, gamma, beta, eps, out, pixels, H, W, C); break;
    default: ln_s2d_kernel<6><<<grid, 256, 0, st>>>(x, gamma, beta, eps, out, pixels, H, W, C); break;
  }
  B200_LAUNCH_OK();
  return B200_OK;
}

// ---- head: spatial mean + LayerNorm ---------------------------------------------------------------------------------
// A block per sample: thread j sums column j over the HW pixels in ascending order (fp32), divides by HW, then the
// block takes the row's mean and variance (warp sums, then the warps' partials in order) and writes LN(m) in fp32.
__global__ void __launch_bounds__(256)
mean_ln_rows_kernel(const __nv_bfloat16* __restrict__ x, int HW, int C, const float* __restrict__ g,
                    const float* __restrict__ be, float eps, float* __restrict__ pooled) {
  extern __shared__ float s_row[];   // [C]
  __shared__ float red[8];
  const int b = blockIdx.x;
  const __nv_bfloat16* src = x + (size_t)b * HW * C;
  float part = 0.f;
  for (int j = threadIdx.x; j < C; j += blockDim.x) {
    float acc = 0.f;
    for (int t = 0; t < HW; t++) acc += __bfloat162float(src[(size_t)t * C + j]);
    s_row[j] = acc / (float)HW;
    part += s_row[j];
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  auto block_total = [&](float v) {
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = 0.f;
    for (int i = 0; i < nw; i++) t += red[i];
    return t;
  };
  const float mean = block_total(part) / (float)C;
  part = 0.f;
  for (int j = threadIdx.x; j < C; j += blockDim.x) {
    const float d = s_row[j] - mean;
    part += d * d;
  }
  const float rstd = rsqrtf(block_total(part) / (float)C + eps);
  for (int j = threadIdx.x; j < C; j += blockDim.x) pooled[(size_t)b * C + j] = (s_row[j] - mean) * rstd * g[j] + be[j];
}

int mean_ln_rows(const __nv_bfloat16* x, int B, int HW, int C, const float* gamma, const float* beta, float eps,
                 float* pooled, cudaStream_t st) {
  B200_CHECK(C >= 1 && C <= 8192 && HW >= 1, B200_ERR_UNSUPPORTED, "mean_ln: C=%d HW=%d", C, HW);
  if (B == 0) return B200_OK;
  mean_ln_rows_kernel<<<B, 256, (size_t)C * sizeof(float), st>>>(x, HW, C, gamma, beta, eps, pooled);
  B200_LAUNCH_OK();
  return B200_OK;
}

}  // namespace b200
