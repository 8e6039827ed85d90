// K4 (SURVEY.md §2.2) on wgmma for head dimension 64 and T <= 320 (every CLIP tower of the benchmark configs but the
// ViT-H/14 image tower, whose head dimension is 80): softmax(Q K^T * hd^-0.5 [+ causal mask]) V per (sample, head).
//
// One CTA = one warpgroup = 64 query rows of one (sample, head).  TMA brings the Q tile and every 64-key block of K
// (boxes of 64 rows x 64 columns of the qkv buffer, 128B swizzle) behind one mbarrier; V is read with ordinary loads
// and written transposed (keys contiguous, same swizzle) so that P.V takes it as a K-major operand, with keys >= T
// zeroed.  Per key block: S = Q K^T (4 x wgmma m64n64k16, both operands in shared memory), mask, online softmax in
// fp32 registers, then O += P V (4 x wgmma m64n64k16 with P as the register A operand: the S accumulator fragment,
// packed to bf16, is exactly the A fragment of the next MMA).  Rows and keys past T of a tile come from the
// neighbouring sample or the TMA zero fill: their scores are masked and their outputs never stored.
#include "embed_kernels.cuh"
#include "gemm.cuh"
#include "ptx.cuh"
#include <atomic>

namespace b200 {

constexpr int ATTW_HD = 64;
constexpr int ATTW_BQ = 64;                        // query rows per CTA
constexpr int ATTW_BK = 64;                        // keys per block
constexpr int ATTW_MAX_T = 320;
constexpr int ATTW_MAX_KB = ATTW_MAX_T / ATTW_BK;  // 5
constexpr int ATTW_TILE = 64 * 128;                // one 64 x 64 bf16 tile, 8 KB
constexpr int ATTW_SMEM = (1 + 2 * ATTW_MAX_KB) * ATTW_TILE + 64 + 1024;

__device__ __forceinline__ uint32_t attw_pack(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

__global__ void __launch_bounds__(128)
attention_wgmma_kernel(const __grid_constant__ CUtensorMap tmQKV, const __nv_bfloat16* __restrict__ qkv,
                       __nv_bfloat16* __restrict__ out, int T, int w, float scale_log2e, int causal) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = ptx::smem_u32(smem_raw);
  uint8_t* base = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* sQ = base;
  uint8_t* sK = base + ATTW_TILE;                          // [kb] tiles: 64 keys x 64 dims
  uint8_t* sVt = sK + ATTW_MAX_KB * ATTW_TILE;             // [kb] tiles: 64 dims x 64 keys
  uint64_t* bar = reinterpret_cast<uint64_t*>(sVt + ATTW_MAX_KB * ATTW_TILE);

  const int q0 = blockIdx.x * ATTW_BQ, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kend = causal ? min(T, q0 + ATTW_BQ) : T;      // keys this tile can see
  const int nkb = (kend + ATTW_BK - 1) / ATTW_BK;
  const int64_t row0 = (int64_t)b * T;

  if (threadIdx.x == 0) {
    ptx::prefetch_tensormap(&tmQKV);
    ptx::mbar_init(bar, 1);
    ptx::fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    ptx::mbar_arrive_expect_tx(bar, (uint32_t)(1 + nkb) * ATTW_TILE);
    ptx::tma_load_2d(sQ, &tmQKV, bar, h * ATTW_HD, (int32_t)(row0 + q0));
    for (int j = 0; j < nkb; j++) ptx::tma_load_2d(sK + j * ATTW_TILE, &tmQKV, bar, w + h * ATTW_HD, (int32_t)(row0 + j * ATTW_BK));
  }
  // V^T: element (dim d, key t) of block t / 64 at row d, 16-byte chunk ((t % 64) / 8) ^ (d % 8), as the 128B swizzle
  // places it; keys >= T are zero (P is 0 there, and 0 * garbage could be NaN)
  const __nv_bfloat16* vbase = qkv + row0 * 3 * w + 2 * w + h * ATTW_HD;
  for (int i = threadIdx.x; i < nkb * ATTW_BK * 8; i += blockDim.x) {
    const int t = i >> 3, c = i & 7;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (t < T) v = *reinterpret_cast<const uint4*>(vbase + (int64_t)t * 3 * w + c * 8);
    const __nv_bfloat16* e = reinterpret_cast<const __nv_bfloat16*>(&v);
    uint8_t* tile = sVt + (t >> 6) * ATTW_TILE;
    const int tk = t & 63;
#pragma unroll
    for (int k = 0; k < 8; k++) {
      const int d = c * 8 + k;
      *reinterpret_cast<__nv_bfloat16*>(tile + d * 128 + ((((tk >> 3) ^ (d & 7)) << 4) | ((tk & 7) << 1))) = e[k];
    }
  }
  ptx::fence_proxy_async();   // generic-proxy writes of V^T -> visible to wgmma
  __syncthreads();
  ptx::mbar_wait(bar, 0);

  // accumulator fragment: register i holds row 16*warp + lane/4 + 8*((i/2)%2), column 8*(i/4) + 2*(lane%4) + i%2
  const int r_lo = q0 + 16 * warp + (lane >> 2), r_hi = r_lo + 8;
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; i++) o[i] = 0.f;
  float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;
  const uint64_t dq = ptx::wgmma_desc_k_sw128(ptx::smem_u32(sQ));

  for (int j = 0; j < nkb; j++) {
    float s[32];
    ptx::wgmma_fence();
    const uint64_t dk = ptx::wgmma_desc_k_sw128(ptx::smem_u32(sK + j * ATTW_TILE));
#pragma unroll
    for (int k = 0; k < ATTW_HD / 16; k++) ptx::wgmma_bf16<64>(s, dq + (uint64_t)(k * 2), dk + (uint64_t)(k * 2), k != 0 ? 1u : 0u);
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_regs(s);

    float bm_lo = -INFINITY, bm_hi = -INFINITY;
#pragma unroll
    for (int i = 0; i < 32; i++) {
      const int key = j * ATTW_BK + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
      const int row = ((i >> 1) & 1) ? r_hi : r_lo;
      if (key >= T || (causal && key > row)) s[i] = -INFINITY;
      if ((i >> 1) & 1) bm_hi = fmaxf(bm_hi, s[i]);
      else bm_lo = fmaxf(bm_lo, s[i]);
    }
    bm_lo = fmaxf(bm_lo, __shfl_xor_sync(0xffffffffu, bm_lo, 1));
    bm_lo = fmaxf(bm_lo, __shfl_xor_sync(0xffffffffu, bm_lo, 2));
    bm_hi = fmaxf(bm_hi, __shfl_xor_sync(0xffffffffu, bm_hi, 1));
    bm_hi = fmaxf(bm_hi, __shfl_xor_sync(0xffffffffu, bm_hi, 2));
    const float mn_lo = fmaxf(m_lo, bm_lo), mn_hi = fmaxf(m_hi, bm_hi);
    // rows that have seen no live key yet keep m = -inf; avoid (-inf) - (-inf)
    const float ms_lo = mn_lo == -INFINITY ? 0.f : mn_lo, ms_hi = mn_hi == -INFINITY ? 0.f : mn_hi;
    const float a_lo = exp2f((m_lo - ms_lo) * scale_log2e), a_hi = exp2f((m_hi - ms_hi) * scale_log2e);
    m_lo = mn_lo;
    m_hi = mn_hi;
    l_lo *= a_lo;
    l_hi *= a_hi;
#pragma unroll
    for (int i = 0; i < 32; i++) {
      const bool hi = (i >> 1) & 1;
      o[i] *= hi ? a_hi : a_lo;
      s[i] = exp2f((s[i] - (hi ? ms_hi : ms_lo)) * scale_log2e);
      if (hi) l_hi += s[i];
      else l_lo += s[i];
    }
    // P as the A operand: k-slice kk covers accumulator column blocks 2kk, 2kk+1
    uint32_t pa[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; kk++) {
      pa[kk][0] = attw_pack(s[8 * kk + 0], s[8 * kk + 1]);
      pa[kk][1] = attw_pack(s[8 * kk + 2], s[8 * kk + 3]);
      pa[kk][2] = attw_pack(s[8 * kk + 4], s[8 * kk + 5]);
      pa[kk][3] = attw_pack(s[8 * kk + 6], s[8 * kk + 7]);
    }
    ptx::wgmma_fence();
    const uint64_t dv = ptx::wgmma_desc_k_sw128(ptx::smem_u32(sVt + j * ATTW_TILE));
#pragma unroll
    for (int kk = 0; kk < 4; kk++) ptx::wgmma_m64n64k16_bf16_rs(o, pa[kk], dv + (uint64_t)(kk * 2), 1u);
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::fence_regs(o);
  }

  l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1);
  l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
  l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
  l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
  const float i_lo = 1.0f / l_lo, i_hi = 1.0f / l_hi;
  __nv_bfloat16* ob = out + row0 * w + h * ATTW_HD;
#pragma unroll
  for (int n = 0; n < 8; n++) {
    const int col = 8 * n + 2 * (lane & 3);
    if (r_lo < T) *reinterpret_cast<uint32_t*>(ob + (int64_t)r_lo * w + col) = attw_pack(o[4 * n] * i_lo, o[4 * n + 1] * i_lo);
    if (r_hi < T) *reinterpret_cast<uint32_t*>(ob + (int64_t)r_hi * w + col) = attw_pack(o[4 * n + 2] * i_hi, o[4 * n + 3] * i_hi);
  }
}

bool attention_wgmma_supported(int T, int heads, int w) {
  return heads > 0 && w == heads * ATTW_HD && T >= 1 && T <= ATTW_MAX_T;
}

int attention_wgmma(const CUtensorMap& tmQKV, const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int T, int heads, int w,
                    int causal, cudaStream_t st) {
  B200_CHECK(attention_wgmma_supported(T, heads, w), B200_ERR_UNSUPPORTED,
             "attention_wgmma: head dim 64 and T <= %d only (T=%d heads=%d w=%d)", ATTW_MAX_T, T, heads, w);
  if (B == 0) return B200_OK;
  static std::atomic<unsigned long long> configured{0};  // bit per device: the attribute is per context
  int dev = 0;
  B200_CUDA(cudaGetDevice(&dev));
  if (!(configured.load() >> (dev & 63) & 1ull)) {
    B200_CUDA(cudaFuncSetAttribute(attention_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATTW_SMEM));
    configured.fetch_or(1ull << (dev & 63));
  }
  const float scale_log2e = 0.125f * 1.4426950408889634f;   // hd^-0.5 * log2(e)
  attention_wgmma_kernel<<<dim3((T + ATTW_BQ - 1) / ATTW_BQ, heads, B), 128, ATTW_SMEM, st>>>(tmQKV, qkv, out, T, w,
                                                                                             scale_log2e, causal);
  B200_LAUNCH_OK();
  return B200_OK;
}

}  // namespace b200
