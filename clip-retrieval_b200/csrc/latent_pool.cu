// SigLIP's latent-query attention pool (timm AttentionPoolLatent with one latent token): the image tower's tokens are
// normed, projected to k | v by a GEMM, and one learned query per head attends over all of them.  The query does not
// depend on the input, so q = q_proj(latent) arrives precomputed (fp32, at load time).  One CTA per (head, sample):
//   1. scores s_t = (q_h . k_{b,t,h}) * hd^-0.5, one thread per key, fp32 dot products in dim order;
//   2. the block maximum m, then p_t = exp(s_t - m) and l = sum_t p_t (fp32, fixed reduction order);
//   3. o_j = (sum_t p_t v_{b,t,h,j}) / l: each thread owns one 16-byte chunk of V columns over a strided slice of
//      the keys, and the slices are added in slice order, so the result is deterministic.
// Every K and V element is read once: the kernel is bound by HBM (T * 2w * 2 bytes per sample).
#include "embed_kernels.cuh"
#include <algorithm>

namespace b200 {

constexpr int LP_THREADS = 256;

__device__ __forceinline__ float lp_block_reduce(float v, float* red, bool is_max) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    const float u = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, u) : v + u;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = red[0];
  for (int i = 1; i < LP_THREADS / 32; i++) t = is_max ? fmaxf(t, red[i]) : t + red[i];
  return t;
}

__global__ void __launch_bounds__(LP_THREADS)
latent_pool_kernel(const __nv_bfloat16* __restrict__ kv, const float* __restrict__ q, __nv_bfloat16* __restrict__ out,
                   int T, int w, int hd, float scale) {
  extern __shared__ float lp_smem[];
  const int cpr = hd / 8;                  // 16-byte chunks per head row
  const int nsl = LP_THREADS / cpr;        // key slices of step 3
  float* s_q = lp_smem;                    // [hd]
  float* s_p = s_q + hd;                   // [T]
  float* s_part = s_p + T;                 // [nsl][hd]
  __shared__ float red[LP_THREADS / 32];
  const int h = blockIdx.x, b = blockIdx.y;
  const size_t ld = (size_t)2 * w;
  const __nv_bfloat16* kb = kv + (size_t)b * T * ld + (size_t)h * hd;
  for (int j = threadIdx.x; j < hd; j += LP_THREADS) s_q[j] = q[h * hd + j];
  __syncthreads();

  float mx = -INFINITY;
  for (int t = threadIdx.x; t < T; t += LP_THREADS) {
    const __nv_bfloat16* kr = kb + (size_t)t * ld;
    float acc = 0.f;
    for (int c = 0; c < cpr; c++) {
      const uint4 u = *reinterpret_cast<const uint4*>(kr + c * 8);
      const __nv_bfloat162* e = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const float2 f = __bfloat1622float2(e[j]);
        acc = fmaf(s_q[c * 8 + 2 * j], f.x, acc);
        acc = fmaf(s_q[c * 8 + 2 * j + 1], f.y, acc);
      }
    }
    const float sc = acc * scale;
    s_p[t] = sc;
    mx = fmaxf(mx, sc);
  }
  mx = lp_block_reduce(mx, red, true);
  float part = 0.f;
  for (int t = threadIdx.x; t < T; t += LP_THREADS) {
    const float p = expf(s_p[t] - mx);
    s_p[t] = p;
    part += p;
  }
  const float l = lp_block_reduce(part, red, false);   // its barriers also publish s_p

  const int slice = threadIdx.x / cpr, c = threadIdx.x - slice * cpr;
  if (slice < nsl) {
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; j++) acc[j] = 0.f;
    const __nv_bfloat16* vb = kb + w + c * 8;
    for (int t = slice; t < T; t += nsl) {
      const uint4 u = *reinterpret_cast<const uint4*>(vb + (size_t)t * ld);
      const __nv_bfloat162* e = reinterpret_cast<const __nv_bfloat162*>(&u);
      const float p = s_p[t];
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const float2 f = __bfloat1622float2(e[j]);
        acc[2 * j] = fmaf(p, f.x, acc[2 * j]);
        acc[2 * j + 1] = fmaf(p, f.y, acc[2 * j + 1]);
      }
    }
#pragma unroll
    for (int j = 0; j < 8; j++) s_part[slice * hd + c * 8 + j] = acc[j];
  }
  __syncthreads();
  const float inv = 1.0f / l;
  for (int j = threadIdx.x; j < hd; j += LP_THREADS) {
    float o = 0.f;
    for (int s = 0; s < nsl; s++) o += s_part[s * hd + j];
    out[(size_t)b * w + h * hd + j] = __float2bfloat16_rn(o * inv);
  }
}

int latent_pool_attention(const __nv_bfloat16* kv, const float* q, __nv_bfloat16* out, int B, int T, int heads, int w,
                          cudaStream_t st) {
  B200_CHECK(heads > 0 && w % heads == 0, B200_ERR_INVALID, "latent_pool: width %d not divisible by heads %d", w, heads);
  const int hd = w / heads;
  B200_CHECK(hd % 8 == 0 && hd <= 128 && T >= 1 && B >= 0 && B <= 65535 && heads <= 65535, B200_ERR_UNSUPPORTED,
             "latent_pool: head dim %d (need a multiple of 8, <= 128), T %d, B %d", hd, T, B);
  if (B == 0) return B200_OK;
  const size_t smem = ((size_t)hd + T + (size_t)(LP_THREADS / (hd / 8)) * hd) * sizeof(float);
  B200_CHECK(smem <= 220 * 1024, B200_ERR_UNSUPPORTED, "latent_pool: %d tokens do not fit in shared memory", T);
  if (smem > 48 * 1024)
    B200_CUDA(cudaFuncSetAttribute(latent_pool_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  latent_pool_kernel<<<dim3(heads, B), LP_THREADS, smem, st>>>(kv, q, out, T, w, hd, 1.0f / sqrtf((float)hd));
  B200_LAUNCH_OK();
  return B200_OK;
}

}  // namespace b200
