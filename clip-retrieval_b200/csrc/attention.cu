// K4 (SURVEY.md §2.2): softmax(Q K^T * hd^-0.5 [+ causal mask]) V per (sample, head), over the fused
// qkv buffer written by the in-proj GEMM.  Small-T regime (T = 50 / 77 / 257): the whole K and V
// of one head sit in shared memory (padded rows, conflict-free ldmatrix), each warp owns 16 query
// rows at a time and runs the flash-style online softmax in fp32 registers.
// First version on mma.sync.m16n8k16 (bf16 in, fp32 accumulate); 4% of the forward's flops.
// Per-sample key lengths (len[b] in 1..T) as in attention_wgmma.cu: keys >= len[b] are staged as zeros and masked,
// the key loop stops at the 32-key block holding len[b] - 1, and rows >= len[b] are written as zeros.
#include "embed_kernels.cuh"

namespace b200 {

__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3,
                                                  uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ uint32_t pack2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

constexpr int ATT_KB = 32;  // keys per inner block

template <int HD>
__global__ void __launch_bounds__(256)
attention_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out, int T, int w, float scale_log2e,
                 int causal, const int* __restrict__ len) {
  constexpr int LDS = HD + 8;  // padded row (elements): 144 B / 176 B rows -> conflict-free ldmatrix
  extern __shared__ __align__(16) unsigned char att_smem[];
  __nv_bfloat16* sK = reinterpret_cast<__nv_bfloat16*>(att_smem);
  const int Tp = (T + ATT_KB - 1) / ATT_KB * ATT_KB;
  __nv_bfloat16* sV = sK + (size_t)Tp * LDS;

  const int h = blockIdx.x, b = blockIdx.y;
  const int L = len != nullptr ? min(max(len[b], 1), T) : T;   // keys of this sample
  const int Lp = (L + ATT_KB - 1) / ATT_KB * ATT_KB;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const size_t ld = (size_t)3 * w;
  const __nv_bfloat16* base = qkv + (size_t)b * T * ld + (size_t)h * HD;

  // stage K and V of this head (zero rows past T)
  constexpr int CPR = HD / 8;  // 16-byte chunks per row
  for (int i = threadIdx.x; i < Tp * CPR; i += blockDim.x) {
    const int t = i / CPR, c = i - t * CPR;
    uint4 kv = make_uint4(0, 0, 0, 0), vv = make_uint4(0, 0, 0, 0);
    if (t < L) {
      kv = *reinterpret_cast<const uint4*>(base + (size_t)t * ld + w + c * 8);
      vv = *reinterpret_cast<const uint4*>(base + (size_t)t * ld + 2 * w + c * 8);
    }
    *reinterpret_cast<uint4*>(sK + (size_t)t * LDS + c * 8) = kv;
    *reinterpret_cast<uint4*>(sV + (size_t)t * LDS + c * 8) = vv;
  }
  __syncthreads();

  const int qblocks = (L + 15) / 16;
  const uint32_t sK_u = (uint32_t)__cvta_generic_to_shared(sK);
  const uint32_t sV_u = (uint32_t)__cvta_generic_to_shared(sV);

  for (int qb = warp; qb < qblocks; qb += nwarps) {
    const int r0 = qb * 16 + (lane >> 2), r1 = r0 + 8;
    // Q fragments straight from global: a[ks] = {Q[r0][k0..], Q[r1][k0..], Q[r0][k0+8..], Q[r1][k0+8..]}
    uint32_t qa[HD / 16][4];
#pragma unroll
    for (int ks = 0; ks < HD / 16; ks++) {
      const int k0 = ks * 16 + (lane & 3) * 2;
      qa[ks][0] = r0 < T ? *reinterpret_cast<const uint32_t*>(base + (size_t)r0 * ld + k0) : 0u;
      qa[ks][1] = r1 < T ? *reinterpret_cast<const uint32_t*>(base + (size_t)r1 * ld + k0) : 0u;
      qa[ks][2] = r0 < T ? *reinterpret_cast<const uint32_t*>(base + (size_t)r0 * ld + k0 + 8) : 0u;
      qa[ks][3] = r1 < T ? *reinterpret_cast<const uint32_t*>(base + (size_t)r1 * ld + k0 + 8) : 0u;
    }
    float o[HD / 8][4];
#pragma unroll
    for (int i = 0; i < HD / 8; i++) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

    const int kend = causal ? min(Lp, (qb * 16 + 16 + ATT_KB - 1) / ATT_KB * ATT_KB) : Lp;
    for (int kb = 0; kb < kend; kb += ATT_KB) {
      float s[ATT_KB / 8][4];
#pragma unroll
      for (int nt = 0; nt < ATT_KB / 8; nt++) {
        s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
        for (int kp = 0; kp < HD / 32; kp++) {
          // four 8x8 blocks of K: keys kb+nt*8.., d = kp*32 + {0,8,16,24}
          uint32_t b0, b1, b2, b3;
          const uint32_t addr = sK_u + (uint32_t)(((kb + nt * 8 + (lane & 7)) * LDS + kp * 32 + (lane >> 3) * 8) * 2);
          ldmatrix_x4(b0, b1, b2, b3, addr);
          mma_bf16_16816(s[nt], qa[kp * 2], b0, b1);
          mma_bf16_16816(s[nt], qa[kp * 2 + 1], b2, b3);
        }
        if constexpr (HD % 32 != 0) {
          // tail k-step (HD = 80): d = HD-16 .. HD-1; only matrices 0,1 are meaningful
          uint32_t b0, b1, b2, b3;
          const int dcol = (HD / 32) * 32 + ((lane >> 3) & 1) * 8;
          const uint32_t addr = sK_u + (uint32_t)(((kb + nt * 8 + (lane & 7)) * LDS + dcol) * 2);
          ldmatrix_x4(b0, b1, b2, b3, addr);
          mma_bf16_16816(s[nt], qa[HD / 16 - 1], b0, b1);
        }
      }
      // mask + block row max (scores stay unscaled; the scale folds into the exp2 argument)
      float bm0 = -INFINITY, bm1 = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < ATT_KB / 8; nt++) {
        const int key = kb + nt * 8 + (lane & 3) * 2;
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const int kk = key + e;
          const bool dead0 = kk >= L || (causal && kk > r0);
          const bool dead1 = kk >= L || (causal && kk > r1);
          if (dead0) s[nt][e] = -INFINITY;
          if (dead1) s[nt][2 + e] = -INFINITY;
          bm0 = fmaxf(bm0, s[nt][e]);
          bm1 = fmaxf(bm1, s[nt][2 + e]);
        }
      }
      bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 1));
      bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 2));
      bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 1));
      bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 2));
      const float mn0 = fmaxf(m0, bm0), mn1 = fmaxf(m1, bm1);
      // rows that have seen no live key yet keep m = -inf; avoid (-inf) - (-inf)
      const float ms0 = mn0 == -INFINITY ? 0.f : mn0, ms1 = mn1 == -INFINITY ? 0.f : mn1;
      const float a0 = exp2f((m0 - ms0) * scale_log2e), a1 = exp2f((m1 - ms1) * scale_log2e);
      m0 = mn0;
      m1 = mn1;
      l0 *= a0;
      l1 *= a1;
#pragma unroll
      for (int i = 0; i < HD / 8; i++) {
        o[i][0] *= a0; o[i][1] *= a0;
        o[i][2] *= a1; o[i][3] *= a1;
      }
      uint32_t pa[ATT_KB / 16][4];
#pragma unroll
      for (int nt = 0; nt < ATT_KB / 8; nt++) {
        const float p0 = exp2f((s[nt][0] - ms0) * scale_log2e), p1 = exp2f((s[nt][1] - ms0) * scale_log2e);
        const float p2 = exp2f((s[nt][2] - ms1) * scale_log2e), p3 = exp2f((s[nt][3] - ms1) * scale_log2e);
        l0 += p0 + p1;
        l1 += p2 + p3;
        pa[nt >> 1][(nt & 1) * 2 + 0] = pack2(p0, p1);
        pa[nt >> 1][(nt & 1) * 2 + 1] = pack2(p2, p3);
      }
      // O += P V : V^T fragments through ldmatrix.trans
#pragma unroll
      for (int kk = 0; kk < ATT_KB / 16; kk++) {
#pragma unroll
        for (int dp = 0; dp < HD / 16; dp++) {
          uint32_t b0, b1, b2, b3;
          const int key = kb + kk * 16 + ((lane >> 3) & 1) * 8 + (lane & 7);
          const int dcol = dp * 16 + (lane >> 4) * 8;
          ldmatrix_x4_trans(b0, b1, b2, b3, sV_u + (uint32_t)((key * LDS + dcol) * 2));
          mma_bf16_16816(o[dp * 2], pa[kk], b0, b1);
          mma_bf16_16816(o[dp * 2 + 1], pa[kk], b2, b3);
        }
      }
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float i0 = 1.0f / l0, i1 = 1.0f / l1;
    __nv_bfloat16* ob = out + (size_t)b * T * w + (size_t)h * HD;
#pragma unroll
    for (int i = 0; i < HD / 8; i++) {
      const int col = i * 8 + (lane & 3) * 2;
      if (r0 < T) *reinterpret_cast<uint32_t*>(ob + (size_t)r0 * w + col) = r0 < L ? pack2(o[i][0] * i0, o[i][1] * i0) : 0u;
      if (r1 < T) *reinterpret_cast<uint32_t*>(ob + (size_t)r1 * w + col) = r1 < L ? pack2(o[i][2] * i1, o[i][3] * i1) : 0u;
    }
  }
  // rows of the 16-row query blocks past the sample's keys (none without lengths)
  __nv_bfloat16* ob = out + (size_t)b * T * w + (size_t)h * HD;
  for (int i = qblocks * 16 * CPR + (int)threadIdx.x; i < T * CPR; i += blockDim.x)
    *reinterpret_cast<uint4*>(ob + (size_t)(i / CPR) * w + (i % CPR) * 8) = make_uint4(0u, 0u, 0u, 0u);
}

template <int HD>
static int launch_attention(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int T, int heads, int w, int causal,
                            cudaStream_t st, const int* len) {
  const int Tp = (T + ATT_KB - 1) / ATT_KB * ATT_KB;
  const size_t smem = (size_t)2 * Tp * (HD + 8) * sizeof(__nv_bfloat16);
  B200_CHECK(smem <= 200 * 1024, B200_ERR_UNSUPPORTED, "attention: sequence length %d too long for the small-T kernel", T);
  auto kern = attention_kernel<HD>;
  if (smem > 48 * 1024) B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const float scale_log2e = (1.0f / sqrtf((float)HD)) * 1.4426950408889634f;
  const int qblocks = (T + 15) / 16;
  const int threads = qblocks >= 8 ? 256 : (qblocks >= 4 ? 128 : 64);
  kern<<<dim3(heads, B), threads, smem, st>>>(qkv, out, T, w, scale_log2e, causal, len);
  B200_LAUNCH_OK();
  return B200_OK;
}

int attention(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int T, int heads, int w, int causal, cudaStream_t st,
              const int* len) {
  B200_CHECK(heads > 0 && w % heads == 0, B200_ERR_INVALID, "attention: width %d not divisible by heads %d", w, heads);
  if (B == 0) return B200_OK;
  const int hd = w / heads;
  if (hd == 64) return launch_attention<64>(qkv, out, B, T, heads, w, causal, st, len);
  if (hd == 80) return launch_attention<80>(qkv, out, B, T, heads, w, causal, st, len);
  if (hd == 96) return launch_attention<96>(qkv, out, B, T, heads, w, causal, st, len);
  if (hd == 128) return launch_attention<128>(qkv, out, B, T, heads, w, causal, st, len);
  set_error("attention: head dimension %d not supported (64, 80, 96, 128)", hd);
  return B200_ERR_UNSUPPORTED;
}

}  // namespace b200
