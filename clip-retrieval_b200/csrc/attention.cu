// K4 (SURVEY.md §2.2): softmax(Q K^T * hd^-0.5 [+ causal mask]) V per (sample, head), over the fused
// qkv buffer written by the in-proj GEMM.  Small-T regime (T = 50 / 77 / 257): the whole K and V
// of one head sit in shared memory (padded rows, conflict-free ldmatrix), each warp owns 16 query
// rows at a time and runs the flash-style online softmax in fp32 registers.
// First version on mma.sync.m16n8k16 (bf16 in, fp32 accumulate); 4% of the forward's flops.
// Per-sample key lengths (len[b] in 1..T) as in attention_wgmma.cu: keys >= len[b] are staged as zeros and masked,
// the key loop stops at the 32-key block holding len[b] - 1, and rows >= len[b] are written as zeros.
// Shapes whose whole-head K + V would pass 200 KB run on attention_stream_kernel below, with the same per-block step.
// Head dims 88 and 104 (ViT-g-14, ViT-bigG-14: HD % 16 == 8) take the same kernels with an 8-wide tail at every step:
// the last Q fragment's upper half is zero registers (columns HD.. of the qkv row are the next head's Q, or K), QK^T
// ends with one 8-dim k-step, P.V with one unpaired n8 tile, and the K/V rows are padded to HD + 16 (att_lds).
#include "embed_kernels.cuh"
#include "ptx.cuh"

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

// Padded K/V row in shared memory (elements): an odd number of 16-byte chunks, so that the 8 rows of an ldmatrix
// 8x8 block fall in distinct bank groups.  HD + 8 for HD % 16 == 0 (144 B / 176 B / 208 B / 272 B rows at 64 / 80 / 96
// / 128), HD + 16 for HD % 16 == 8 (208 B / 240 B at 88 / 104; HD + 8 would give an even 12 / 14 chunks).
__host__ __device__ constexpr int att_lds(int hd) { return hd % 16 == 0 ? hd + 8 : hd + 16; }
// k16 Q fragments per row pair: the last one of HD % 16 == 8 holds dims HD-8..HD-1 and zero registers above.
__host__ __device__ constexpr int att_qfrags(int hd) { return (hd + 15) / 16; }

// Q fragments of rows r0 / r1 straight from global (rows >= T read as zeros):
// a[ks] = {Q[r0][k0..], Q[r1][k0..], Q[r0][k0+8..], Q[r1][k0+8..]}; for HD % 16 == 8 the last fragment's upper half
// (dims HD..HD+7, which belong to the next head) is zero and is not loaded.
template <int HD>
__device__ __forceinline__ void load_q_frags(const __nv_bfloat16* base, size_t ld, int r0, int r1, int T, int lane,
                                             uint32_t (&qa)[att_qfrags(HD)][4]) {
#pragma unroll
  for (int ks = 0; ks < HD / 16; ks++) {
    const int k0 = ks * 16 + (lane & 3) * 2;
    qa[ks][0] = r0 < T ? *reinterpret_cast<const uint32_t*>(base + (size_t)r0 * ld + k0) : 0u;
    qa[ks][1] = r1 < T ? *reinterpret_cast<const uint32_t*>(base + (size_t)r1 * ld + k0) : 0u;
    qa[ks][2] = r0 < T ? *reinterpret_cast<const uint32_t*>(base + (size_t)r0 * ld + k0 + 8) : 0u;
    qa[ks][3] = r1 < T ? *reinterpret_cast<const uint32_t*>(base + (size_t)r1 * ld + k0 + 8) : 0u;
  }
  if constexpr (HD % 16 == 8) {
    const int k0 = HD - 8 + (lane & 3) * 2;
    qa[HD / 16][0] = r0 < T ? *reinterpret_cast<const uint32_t*>(base + (size_t)r0 * ld + k0) : 0u;
    qa[HD / 16][1] = r1 < T ? *reinterpret_cast<const uint32_t*>(base + (size_t)r1 * ld + k0) : 0u;
    qa[HD / 16][2] = 0u;
    qa[HD / 16][3] = 0u;
  }
}

// o / l of rows r0 / r1 into ob (the head's column block of the sample's output rows): rows >= L as zeros, rows >= T
// not written.
template <int HD>
__device__ __forceinline__ void store_rows(__nv_bfloat16* ob, int w, int r0, int r1, int T, int L,
                                           const float (&o)[HD / 8][4], float l0, float l1, int lane) {
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.0f / l0, i1 = 1.0f / l1;
#pragma unroll
  for (int i = 0; i < HD / 8; i++) {
    const int col = i * 8 + (lane & 3) * 2;
    if (r0 < T) *reinterpret_cast<uint32_t*>(ob + (size_t)r0 * w + col) = r0 < L ? pack2(o[i][0] * i0, o[i][1] * i0) : 0u;
    if (r1 < T) *reinterpret_cast<uint32_t*>(ob + (size_t)r1 * w + col) = r1 < L ? pack2(o[i][2] * i1, o[i][3] * i1) : 0u;
  }
}

// One 32-key block kb of a warp's 16 query rows (r0 = its row of lane / 4, r1 = r0 + 8): S = Q K^T on mma.sync, the
// mask (keys >= L, and keys > row when causal), the fp32 online softmax update of (m, l, o), then O += P V with P in
// bf16.  sK_u / sV_u address key kb at sK_u + kb * LDS * 2: both kernels call this, the whole-K/V kernel with its
// buffer's base, the streaming kernel with a ring stage's base shifted back by the stage's first key.
template <int HD>
__device__ __forceinline__ void attention_block_step(uint32_t sK_u, uint32_t sV_u, int kb,
                                                     const uint32_t (&qa)[att_qfrags(HD)][4], float (&o)[HD / 8][4],
                                                     float& m0, float& m1, float& l0, float& l1, int r0, int r1, int L,
                                                     int causal, float scale_log2e, int lane) {
  constexpr int LDS = att_lds(HD);
  float s[ATT_KB / 8][4];
  // HD % 16 == 8: K dims HD-8..HD-1 of the block's 32 keys, one 8x8 matrix per 8 keys (matrix nt = keys kb + nt*8..)
  uint32_t kt[4] = {0u, 0u, 0u, 0u};
  if constexpr (HD % 16 == 8)
    ldmatrix_x4(kt[0], kt[1], kt[2], kt[3], sK_u + (uint32_t)(((kb + lane) * LDS + HD - 8) * 2));
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
    if constexpr (HD % 32 >= 16) {
      // 16-wide tail k-step (HD = 80, 88): d = (HD/32)*32 .. +15; only matrices 0,1 are meaningful
      uint32_t b0, b1, b2, b3;
      const int dcol = (HD / 32) * 32 + ((lane >> 3) & 1) * 8;
      const uint32_t addr = sK_u + (uint32_t)(((kb + nt * 8 + (lane & 7)) * LDS + dcol) * 2);
      ldmatrix_x4(b0, b1, b2, b3, addr);
      mma_bf16_16816(s[nt], qa[(HD / 32) * 2], b0, b1);
    }
    if constexpr (HD % 16 == 8) {
      // 8-wide tail k-step (HD = 88, 104): d = HD-8 .. HD-1 against the zero-topped last Q fragment; the K operand's
      // upper half is a zero register too, so the shared-memory padding never enters the sum
      mma_bf16_16816(s[nt], qa[HD / 16], kt[nt], 0u);
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
  if constexpr (HD % 16 == 8) {
    // the unpaired last n8 tile (d = HD-8 .. HD-1): V^T of keys kb + 8j.. as matrix j, so {b0, b1} / {b2, b3} are
    // the k16 halves of keys kb.. / kb+16..
    uint32_t b0, b1, b2, b3;
    ldmatrix_x4_trans(b0, b1, b2, b3, sV_u + (uint32_t)(((kb + lane) * LDS + HD - 8) * 2));
    mma_bf16_16816(o[HD / 8 - 1], pa[0], b0, b1);
    mma_bf16_16816(o[HD / 8 - 1], pa[1], b2, b3);
  }
}

template <int HD>
__global__ void __launch_bounds__(256)
attention_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out, int T, int w, float scale_log2e,
                 int causal, const int* __restrict__ len) {
  constexpr int LDS = att_lds(HD);  // padded row (elements) -> conflict-free ldmatrix
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
    uint32_t qa[att_qfrags(HD)][4];
    load_q_frags<HD>(base, ld, r0, r1, T, lane, qa);
    float o[HD / 8][4];
#pragma unroll
    for (int i = 0; i < HD / 8; i++) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

    const int kend = causal ? min(Lp, (qb * 16 + 16 + ATT_KB - 1) / ATT_KB * ATT_KB) : Lp;
    for (int kb = 0; kb < kend; kb += ATT_KB) {
      attention_block_step<HD>(sK_u, sV_u, kb, qa, o, m0, m1, l0, l1, r0, r1, L, causal, scale_log2e, lane);
    }
    store_rows<HD>(out + (size_t)b * T * w + (size_t)h * HD, w, r0, r1, T, L, o, l0, l1, lane);
  }
  // rows of the 16-row query blocks past the sample's keys (none without lengths)
  __nv_bfloat16* ob = out + (size_t)b * T * w + (size_t)h * HD;
  for (int i = qblocks * 16 * CPR + (int)threadIdx.x; i < T * CPR; i += blockDim.x)
    *reinterpret_cast<uint4*>(ob + (size_t)(i / CPR) * w + (i % CPR) * 8) = make_uint4(0u, 0u, 0u, 0u);
}

// Longer sequences (whole-head K + V past 200 KB of shared memory: T > 704 / 576 / 480 / 352 at head dim 64 / 80 /
// 96 / 128): one CTA per (128-row query chunk, head, sample), chunk fastest so that the chunks of a head read its K/V
// from L2.  Eight warps own 16 query rows each; K and V pass through a ring of ATS_STAGES blocks of 64 keys, filled
// by warp 0 with one bulk copy per row (rows padded to att_lds(HD) elements as above) and handed over by full / empty
// mbarriers, so shared memory no longer grows with T.  The arithmetic per 32-key block is attention_block_step.
// A chunk loads keys < len[b] only, and with causal only keys up to its last row; a chunk wholly at or past len[b]
// writes zeros and loads nothing.
constexpr int ATS_ROWS = 128;    // query rows per CTA (8 warps x 16)
constexpr int ATS_KEYS = 64;     // keys per ring stage
constexpr int ATS_STAGES = 3;

template <int HD>
constexpr size_t attention_stream_smem() {
  return (size_t)ATS_STAGES * 2 * ATS_KEYS * att_lds(HD) * sizeof(__nv_bfloat16) + 2 * ATS_STAGES * sizeof(uint64_t);
}

template <int HD>
__global__ void __launch_bounds__(256, HD <= 96 ? 2 : 1)
attention_stream_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out, int T, int w,
                        float scale_log2e, int causal, const int* __restrict__ len) {
  constexpr int LDS = att_lds(HD);
  constexpr int CPR = HD / 8;                                    // 16-byte chunks per row
  constexpr uint32_t MAT = ATS_KEYS * LDS * sizeof(__nv_bfloat16);   // one stage's K (or V) block, bytes
  constexpr uint32_t STAGE = 2 * MAT;
  extern __shared__ __align__(16) unsigned char att_smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(att_smem + ATS_STAGES * STAGE);
  uint64_t* empty = full + ATS_STAGES;

  const int chunk = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int L = len != nullptr ? min(max(len[b], 1), T) : T;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t ld = (size_t)3 * w;
  const __nv_bfloat16* base = qkv + (size_t)b * T * ld + (size_t)h * HD;
  __nv_bfloat16* ob = out + (size_t)b * T * w + (size_t)h * HD;
  const int row0 = chunk * ATS_ROWS;
  if (row0 >= L) {
    for (int i = threadIdx.x; i < min(ATS_ROWS, T - row0) * CPR; i += blockDim.x)
      *reinterpret_cast<uint4*>(ob + (size_t)(row0 + i / CPR) * w + (i % CPR) * 8) = make_uint4(0u, 0u, 0u, 0u);
    return;
  }
  const int nkeys = causal ? min(L, row0 + ATS_ROWS) : L;       // keys this chunk reads: rows < nkeys of the sample
  const int nblk = (nkeys + ATS_KEYS - 1) / ATS_KEYS;
  const int nlive = min(ATS_ROWS / 16, (L - row0 + 15) / 16);   // warps with a row < L; they alone take part
  if (threadIdx.x == 0) {
    for (int s = 0; s < ATS_STAGES; s++) {
      ptx::mbar_init(&full[s], 1);
      ptx::mbar_init(&empty[s], nlive);
    }
    ptx::fence_barrier_init();
  }
  // The last block's rows >= nkeys are never loaded but are read by its 32-key steps (masked: P = 0).  Zero them in
  // the stage it lands in, so that P . V never meets uninitialised shared memory; an earlier block of the same stage
  // leaves finite K/V rows there instead.
  {
    const int rem = nkeys - (nblk - 1) * ATS_KEYS;
    unsigned char* st = att_smem + ((nblk - 1) % ATS_STAGES) * STAGE;
    for (int i = threadIdx.x; i < (ATS_KEYS - rem) * CPR * 2; i += blockDim.x) {
      const int r = rem + i / (2 * CPR), c = i % (2 * CPR);
      *reinterpret_cast<uint4*>(st + (c / CPR) * MAT + (size_t)r * LDS * 2 + (c % CPR) * 16) = make_uint4(0u, 0u, 0u, 0u);
    }
    ptx::fence_proxy_async();
  }
  __syncthreads();

  const uint32_t ring = ptx::smem_u32(att_smem);
  // warp 0: K and V rows of key block j into stage j % ATS_STAGES
  auto load_block = [&](int j) {
    const int s = j % ATS_STAGES, k0 = j * ATS_KEYS, n = min(ATS_KEYS, nkeys - k0);
    if (lane == 0) ptx::mbar_arrive_expect_tx(&full[s], (uint32_t)n * 2 * HD * sizeof(__nv_bfloat16));
    __syncwarp();
    for (int r = lane; r < n; r += 32) {
      const __nv_bfloat16* src = base + (size_t)(k0 + r) * ld + w;
      const uint32_t dst = ring + s * STAGE + r * LDS * sizeof(__nv_bfloat16);
      ptx::bulk_load(dst, src, HD * sizeof(__nv_bfloat16), &full[s]);
      ptx::bulk_load(dst + MAT, src + w, HD * sizeof(__nv_bfloat16), &full[s]);
    }
  };
  if (warp == 0)
    for (int j = 0; j < min(ATS_STAGES - 1, nblk); j++) load_block(j);

  const int qb = chunk * (ATS_ROWS / 16) + warp;
  if (warp < nlive) {
    const int r0 = qb * 16 + (lane >> 2), r1 = r0 + 8;
    uint32_t qa[att_qfrags(HD)][4];
    load_q_frags<HD>(base, ld, r0, r1, T, lane, qa);
    float o[HD / 8][4];
#pragma unroll
    for (int i = 0; i < HD / 8; i++) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    const int Lp = (L + ATT_KB - 1) / ATT_KB * ATT_KB;
    const int kend = causal ? min(Lp, (qb * 16 + 16 + ATT_KB - 1) / ATT_KB * ATT_KB) : Lp;
    for (int j = 0; j < nblk; j++) {
      // refill the stage block j - 1 used, once every live warp is done with it
      if (warp == 0 && j + ATS_STAGES - 1 < nblk) {
        if (j > 0) ptx::mbar_wait(&empty[(j - 1) % ATS_STAGES], ((j - 1) / ATS_STAGES) & 1);
        load_block(j + ATS_STAGES - 1);
      }
      const int s = j % ATS_STAGES;
      ptx::mbar_wait(&full[s], (j / ATS_STAGES) & 1);
      // key kb of block j sits at row kb - j * ATS_KEYS of the stage
      const uint32_t sK_u = ring + s * STAGE - (uint32_t)(j * ATS_KEYS * LDS * sizeof(__nv_bfloat16));
      for (int kb = j * ATS_KEYS; kb < min(kend, (j + 1) * ATS_KEYS); kb += ATT_KB)
        attention_block_step<HD>(sK_u, sK_u + MAT, kb, qa, o, m0, m1, l0, l1, r0, r1, L, causal, scale_log2e, lane);
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(&empty[s]);
    }
    store_rows<HD>(ob, w, r0, r1, T, L, o, l0, l1, lane);
  } else {
    // rows of this warp lie at or past len[b]
    for (int i = lane; i < max(0, min(16, T - qb * 16)) * CPR; i += 32)
      *reinterpret_cast<uint4*>(ob + (size_t)(qb * 16 + i / CPR) * w + (i % CPR) * 8) = make_uint4(0u, 0u, 0u, 0u);
  }
}

template <int HD>
static int launch_attention_stream(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int T, int heads, int w,
                                   int causal, cudaStream_t st, const int* len) {
  B200_CHECK(B <= 65535 && heads <= 65535, B200_ERR_UNSUPPORTED,
             "attention: %d samples x %d heads at sequence length %d: the streaming kernel takes at most 65535 of each",
             B, heads, T);
  constexpr size_t smem = attention_stream_smem<HD>();
  auto kern = attention_stream_kernel<HD>;
  B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const float scale_log2e = (1.0f / sqrtf((float)HD)) * 1.4426950408889634f;
  kern<<<dim3((T + ATS_ROWS - 1) / ATS_ROWS, heads, B), 256, smem, st>>>(qkv, out, T, w, scale_log2e, causal, len);
  B200_LAUNCH_OK();
  return B200_OK;
}

template <int HD>
static int launch_attention(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int T, int heads, int w, int causal,
                            cudaStream_t st, const int* len) {
  const int Tp = (T + ATT_KB - 1) / ATT_KB * ATT_KB;
  const size_t smem = (size_t)2 * Tp * att_lds(HD) * sizeof(__nv_bfloat16);
  if (smem > 200 * 1024) return launch_attention_stream<HD>(qkv, out, B, T, heads, w, causal, st, len);
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
  if (hd == 88) return launch_attention<88>(qkv, out, B, T, heads, w, causal, st, len);
  if (hd == 96) return launch_attention<96>(qkv, out, B, T, heads, w, causal, st, len);
  if (hd == 104) return launch_attention<104>(qkv, out, B, T, heads, w, causal, st, len);
  if (hd == 128) return launch_attention<128>(qkv, out, B, T, heads, w, causal, st, len);
  set_error("attention: head dimension %d not supported (64, 80, 88, 96, 104, 128)", hd);
  return B200_ERR_UNSUPPORTED;
}

}  // namespace b200
