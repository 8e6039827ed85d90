// K4 (SURVEY.md §2.2) on wgmma for head dimension 64 and T <= 320 (every CLIP tower of the benchmark configs but the
// ViT-H/14 image tower, whose head dimension is 80): softmax(Q K^T * hd^-0.5 [+ causal mask]) V per (sample, head).
//
// One CTA = one (sample, head), two consumer warpgroups.  At the start one thread issues every TMA load of the head:
// the first Q tile of each warpgroup, then K and V block by block (64 keys x 64 dims each, 128B swizzle, one mbarrier
// per block so that the first Q K^T waits for K_0 alone), then the second Q tile of each warpgroup.  The map is 3-D over
// (column, token, sample) and clipped at T, so rows >= T of every box are zeros: the next sample is never read.
// Warpgroup g takes query tiles g, g + 2, g + 4 (64 rows each) from two Q slots; when the last Q K^T of a tile has
// completed, the slot is refilled with the tile after next.  K and V are read once per (sample, head) and stay in shared
// memory for every query tile.
//
// Per key block j of a query tile: S = Q K^T (4 x wgmma m64nNk16, both operands in shared memory), online softmax in
// fp32 registers, then O += P V (wgmma m64n64k16 with P as the register A operand -- the S accumulator fragment packed
// to bf16 is exactly the A fragment -- and V as the MN-major B operand straight from its TMA tile).  P_j V_j and
// S_{j+1} are issued back to back after the softmax of block j, and the warpgroup waits for both before the next
// softmax: inside one warpgroup the exponentials never overlap its own wgmmas, only those of the other warpgroups on the
// SM (two CTAs of two).  Only the last key block of a tile (the end of the sequence, or the causal diagonal) is masked,
// and it is computed on N = 16 * ceil(keys / 16) columns, its softmax on those columns and as many k16 steps of P V.
//
// The exponentials are ex2.approx.ftz: the same MUFU result as exp2f except that results below 2^-126 are flushed to
// zero, which saves the range test and rescale exp2f wraps around every score.
//
// With per-sample key lengths (len[b] in 1..T, the key-padding mask of a bidirectional encoder) a sample sees keys
// < len[b] only: the key blocks at or past len[b] are not loaded, the query tiles wholly past it are not computed, and
// every row >= len[b] of the output is written as zeros.  len == nullptr is len[b] = T, and then the arithmetic and the
// stores are the ones of the kernel without lengths.
#include "embed_kernels.cuh"
#include "gemm.cuh"
#include "ptx.cuh"
#include <atomic>

namespace b200 {

constexpr int ATTW_HD = 64;
constexpr int ATTW_BQ = 64;                        // query rows per tile
constexpr int ATTW_BK = 64;                        // keys per block
constexpr int ATTW_MAX_T = 320;
constexpr int ATTW_MAX_KB = ATTW_MAX_T / ATTW_BK;  // 5
constexpr int ATTW_TILE = 64 * 128;                // one 64 x 64 bf16 tile, 8 KB
constexpr int ATTW_QSLOTS = 4;                     // two Q tiles per consumer warpgroup
constexpr int ATTW_THREADS = 256;
// barriers: K blocks, V blocks, Q slots
constexpr int ATTW_NBAR = 2 * ATTW_MAX_KB + ATTW_QSLOTS;
constexpr int ATTW_BAR_BYTES = 8 * ATTW_NBAR;

// K and V of every key block plus the Q slots, and 1 KB to align the tiles.  The barriers live in that alignment gap
// when it is large enough, else after the tiles: at T = 320 this is 115 712 B, so two CTAs share an SM.
static int attw_smem_bytes(int T) {
  return (2 * ((T + ATTW_BK - 1) / ATTW_BK) + ATTW_QSLOTS) * ATTW_TILE + 1024;
}

__device__ __forceinline__ uint32_t attw_pack(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

// S = Q K^T of one key block on `cols` (16, 32, 48 or 64) columns; accumulator registers past cols / 2 are not written.
__device__ __forceinline__ void attw_qk(float (&s)[32], uint64_t dq, uint64_t dk, int cols) {
  ptx::wgmma_fence();
#pragma unroll
  for (int k = 0; k < ATTW_HD / 16; k++) {
    const uint64_t a = dq + (uint64_t)(k * 2), b = dk + (uint64_t)(k * 2);
    const uint32_t acc = k != 0 ? 1u : 0u;
    if (cols == 64) ptx::wgmma_m64n64k16_bf16(s, a, b, acc);
    else if (cols == 48) ptx::wgmma_m64n48k16_bf16(*reinterpret_cast<float(*)[24]>(&s[0]), a, b, acc);
    else if (cols == 32) ptx::wgmma_m64n32k16_bf16(*reinterpret_cast<float(*)[16]>(&s[0]), a, b, acc);
    else ptx::wgmma_m64n16k16_bf16(*reinterpret_cast<float(*)[8]>(&s[0]), a, b, acc);
  }
  ptx::wgmma_commit();
}

struct AttwRow {
  float m_lo, m_hi, l_lo, l_hi;
};

// Online softmax of one score block (in place: s becomes P, unnormalised), the matching rescale of O, and P packed to
// bf16 as the A operand of P V (k-slice kk covers accumulator column blocks 2kk, 2kk+1).  Only the first NREG
// registers (NREG / 2 columns) are computed: the last block of a tile is narrowed to 16 * ceil(keys / 16) columns, and
// the registers past them would only be masked to -inf, giving P = 0 that no k16 step of P V reads.  Leaving them out
// changes no maximum and no sum.
// accumulator fragment: register i holds row 16*warp + lane/4 + 8*((i/2)%2), column 8*(i/4) + 2*(lane%4) + i%2
template <bool MASK, int NREG>
__device__ __forceinline__ void attw_softmax(float (&s)[32], float (&o)[32], uint32_t (&pa)[4][4], AttwRow& r,
                                             int lane, int key0, int kend, int r_lo, int causal, float scale_log2e) {
  float bm_lo = -INFINITY, bm_hi = -INFINITY;
#pragma unroll
  for (int i = 0; i < NREG; i++) {
    if (MASK) {
      const int key = key0 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
      const int row = r_lo + 8 * ((i >> 1) & 1);
      if (key >= kend || (causal && key > row)) s[i] = -INFINITY;
    }
    if ((i >> 1) & 1) bm_hi = fmaxf(bm_hi, s[i]);
    else bm_lo = fmaxf(bm_lo, s[i]);
  }
  bm_lo = fmaxf(bm_lo, __shfl_xor_sync(0xffffffffu, bm_lo, 1));
  bm_lo = fmaxf(bm_lo, __shfl_xor_sync(0xffffffffu, bm_lo, 2));
  bm_hi = fmaxf(bm_hi, __shfl_xor_sync(0xffffffffu, bm_hi, 1));
  bm_hi = fmaxf(bm_hi, __shfl_xor_sync(0xffffffffu, bm_hi, 2));
  const float mn_lo = fmaxf(r.m_lo, bm_lo), mn_hi = fmaxf(r.m_hi, bm_hi);
  // rows that have seen no live key yet keep m = -inf; avoid (-inf) - (-inf)
  const float ms_lo = mn_lo == -INFINITY ? 0.f : mn_lo, ms_hi = mn_hi == -INFINITY ? 0.f : mn_hi;
  const float a_lo = ptx::ex2_ftz((r.m_lo - ms_lo) * scale_log2e), a_hi = ptx::ex2_ftz((r.m_hi - ms_hi) * scale_log2e);
  r.m_lo = mn_lo;
  r.m_hi = mn_hi;
  r.l_lo *= a_lo;
  r.l_hi *= a_hi;
#pragma unroll
  for (int i = 0; i < 32; i++) {
    const bool hi = (i >> 1) & 1;
    o[i] *= hi ? a_hi : a_lo;
    if (i >= NREG) continue;
    // (s - m) * scale rounded as written, not fused into one fma: P, and so every embedding, stays bit for bit what
    // the earlier one-tile-per-CTA kernel computed
    s[i] = ptx::ex2_ftz((s[i] - (hi ? ms_hi : ms_lo)) * scale_log2e);
    if (hi) r.l_hi += s[i];
    else r.l_lo += s[i];
  }
#pragma unroll
  for (int kk = 0; kk < 4; kk++) {
    pa[kk][0] = kk < NREG / 8 ? attw_pack(s[8 * kk + 0], s[8 * kk + 1]) : 0u;
    pa[kk][1] = kk < NREG / 8 ? attw_pack(s[8 * kk + 2], s[8 * kk + 3]) : 0u;
    pa[kk][2] = kk < NREG / 8 ? attw_pack(s[8 * kk + 4], s[8 * kk + 5]) : 0u;
    pa[kk][3] = kk < NREG / 8 ? attw_pack(s[8 * kk + 6], s[8 * kk + 7]) : 0u;
  }
}

// 4 x 4 transpose of 32-bit words across the lanes of a quad: lane q returns, in b[k], word q of lane k's a[].
__device__ __forceinline__ void attw_quad_transpose(const uint32_t (&a)[4], uint32_t (&b)[4], int q) {
#pragma unroll
  for (int k = 0; k < 4; k++) b[k] = a[k];
#pragma unroll
  for (int x = 1; x < 4; x++) {
    const int p = q ^ x;   // partner lane in the quad: it wants my a[p], I want its a[q]
    const uint32_t send = p == 0 ? a[0] : p == 1 ? a[1] : p == 2 ? a[2] : a[3];
    const uint32_t got = __shfl_xor_sync(0xffffffffu, send, x);
#pragma unroll
    for (int k = 0; k < 4; k++)
      if (k == p) b[k] = got;
  }
}

__global__ void __launch_bounds__(ATTW_THREADS, 2)
attention_wgmma_kernel(const __grid_constant__ CUtensorMap tmQKV, __nv_bfloat16* __restrict__ out, int T, int w,
                       float scale_log2e, int causal, const int* __restrict__ len) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t pad = (1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u;
  uint8_t* base = smem_raw + pad;
  const int nkb = (T + ATTW_BK - 1) / ATTW_BK;      // key blocks of the head; also its query tiles
  uint8_t* sK = base;                                // [nkb] 64 keys x 64 dims
  uint8_t* sV = sK + nkb * ATTW_TILE;                // [nkb] 64 keys x 64 dims
  uint8_t* sQ = sV + nkb * ATTW_TILE;                // [ATTW_QSLOTS]: slots 2g, 2g + 1 belong to warpgroup g
  uint64_t* bar = reinterpret_cast<uint64_t*>(pad >= (uint32_t)ATTW_BAR_BYTES ? smem_raw : sQ + ATTW_QSLOTS * ATTW_TILE);
  uint64_t* barK = bar;
  uint64_t* barV = bar + ATTW_MAX_KB;
  uint64_t* barQ = bar + 2 * ATTW_MAX_KB;

  const int h = blockIdx.x, b = blockIdx.y;
  const int L = len != nullptr ? min(max(len[b], 1), T) : T;   // keys of this sample
  const int nlb = (L + ATTW_BK - 1) / ATTW_BK;      // key blocks loaded and query tiles computed
  // the warpgroup index through a shuffle: the compiler then knows it is uniform across the warp, and so is every
  // branch around a wgmma that depends on it (else it serialises the wgmmas)
  const int wg = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 7, 0);
  const int tid = threadIdx.x & 127, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
  const int cq = h * ATTW_HD, ck = w + h * ATTW_HD, cv = 2 * w + h * ATTW_HD;
  // query tile t: warpgroup t % 2, its (t / 2)-th tile, in slot 2 (t % 2) + (t / 2) % 2, phase (t / 4) % 2
  auto load_q = [&](int t) {
    const int slot = 2 * (t & 1) + ((t >> 1) & 1);
    ptx::mbar_arrive_expect_tx(barQ + slot, ATTW_TILE);
    ptx::tma_load_3d(sQ + slot * ATTW_TILE, &tmQKV, barQ + slot, cq, t * ATTW_BQ, b);
  };

  if (threadIdx.x == 0) {
    ptx::prefetch_tensormap(&tmQKV);
    for (int i = 0; i < ATTW_NBAR; i++) ptx::mbar_init(bar + i, 1);
    ptx::fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    load_q(0);
    if (nlb > 1) load_q(1);
    for (int j = 0; j < nlb; j++) {
      ptx::mbar_arrive_expect_tx(barK + j, ATTW_TILE);
      ptx::tma_load_3d(sK + j * ATTW_TILE, &tmQKV, barK + j, ck, j * ATTW_BK, b);
      ptx::mbar_arrive_expect_tx(barV + j, ATTW_TILE);
      ptx::tma_load_3d(sV + j * ATTW_TILE, &tmQKV, barV + j, cv, j * ATTW_BK, b);
    }
    for (int t = 2; t < nlb && t < ATTW_QSLOTS; t++) load_q(t);
  }

  __nv_bfloat16* ob = out + (int64_t)b * T * w + h * ATTW_HD;
  for (int t = wg; t < nlb; t += 2) {
    const int slot = 2 * wg + ((t >> 1) & 1);
    const int q0 = t * ATTW_BQ;
    const int kend = causal ? min(L, q0 + ATTW_BQ) : L;       // keys this tile can see
    const int nkt = (kend + ATTW_BK - 1) / ATTW_BK;
    const int last_cols = 16 * ((kend - (nkt - 1) * ATTW_BK + 15) / 16);
    const int r_lo = q0 + 16 * warp + (lane >> 2);
    // a warp whose 16 rows all lie at or past the sample's keys (warps 1-3 of the last tile at T = 257) has no output
    // to compute: it skips the softmax and the stores, and takes part in every wgmma of its warpgroup with P = 0
    const bool live = q0 + 16 * warp < L;
    ptx::mbar_wait(barQ + slot, (t >> 2) & 1);
    const uint64_t dq = ptx::wgmma_desc_k_sw128(ptx::smem_u32(sQ + slot * ATTW_TILE));

    float o[32];
#pragma unroll
    for (int i = 0; i < 32; i++) o[i] = 0.f;
    ptx::fence_regs(o);   // zeroed before S_0 is issued, not in the middle of the wgmma pipeline
    AttwRow r{-INFINITY, -INFINITY, 0.f, 0.f};
    float s[32];

    auto issue_s = [&](int j) {
      ptx::mbar_wait(barK + j, 0);
      attw_qk(s, dq, ptx::wgmma_desc_k_sw128(ptx::smem_u32(sK + j * ATTW_TILE)), j == nkt - 1 ? last_cols : 64);
      ptx::fence_regs(s);
    };
    // block j: S_j and P_{j-1} V_{j-1} are in flight.  Once they are done: softmax of block j, then O += P_j V_j and
    // S_{j+1} = Q K_{j+1}^T go to the tensor cores back to back (S is free once P_j is packed)
    auto block = [&](int j) {
      const bool last = j == nkt - 1;
      ptx::wgmma_wait<0>();
      ptx::fence_regs(s);
      ptx::fence_regs(o);
      if (last) {
        // the tile's last Q K^T is done: once every warp of the warpgroup is here, the Q slot can be refilled
        ptx::named_barrier_sync(1 + wg, 128);
        if (tid == 0 && t + ATTW_QSLOTS < nlb) load_q(t + ATTW_QSLOTS);
      }
      uint32_t pa[4][4];
      if (live) {
        const int key0 = j * ATTW_BK;
        if (!last) attw_softmax<false, 32>(s, o, pa, r, lane, key0, kend, r_lo, causal, scale_log2e);
        else if (last_cols == 16) attw_softmax<true, 8>(s, o, pa, r, lane, key0, kend, r_lo, causal, scale_log2e);
        else if (last_cols == 32) attw_softmax<true, 16>(s, o, pa, r, lane, key0, kend, r_lo, causal, scale_log2e);
        else if (last_cols == 48) attw_softmax<true, 24>(s, o, pa, r, lane, key0, kend, r_lo, causal, scale_log2e);
        else attw_softmax<true, 32>(s, o, pa, r, lane, key0, kend, r_lo, causal, scale_log2e);
      } else {
#pragma unroll
        for (int kk = 0; kk < 4; kk++) pa[kk][0] = pa[kk][1] = pa[kk][2] = pa[kk][3] = 0u;
      }
      const int ksteps = last ? last_cols / 16 : 4;
      ptx::mbar_wait(barV + j, 0);
      ptx::wgmma_fence();
      const uint64_t dv = ptx::wgmma_desc_mn_sw128(ptx::smem_u32(sV + j * ATTW_TILE));
#pragma unroll
      for (int kk = 0; kk < 4; kk++)
        if (kk < ksteps) ptx::wgmma_m64n64k16_bf16_rs_tb(o, pa[kk], dv + (uint64_t)kk * ptx::WGMMA_DESC_MN_SW128_K16, 1u);
      ptx::wgmma_commit();
      ptx::fence_regs(o);
      if (!last) issue_s(j + 1);
    };

    issue_s(0);
#pragma unroll 1
    for (int j = 0; j < nkt; j++) block(j);
    ptx::wgmma_wait<0>();
    ptx::fence_regs(o);
    if (!live) continue;

    float l_lo = r.l_lo, l_hi = r.l_hi;
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1);
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
    const float i_lo = 1.0f / l_lo, i_hi = 1.0f / l_hi;
    // 16-byte stores: the quad of lanes holding a row exchanges words so that lane q owns columns 8q..8q+7 and
    // 32+8q..32+8q+7 of both its rows
    const int q = lane & 3;
#pragma unroll
    for (int half = 0; half < 2; half++) {
      const int row = r_lo + 8 * half;
      const float inv = half ? i_hi : i_lo;
#pragma unroll
      for (int g = 0; g < 2; g++) {
        uint32_t a[4], c[4];
#pragma unroll
        for (int k = 0; k < 4; k++) a[k] = attw_pack(o[4 * (4 * g + k) + 2 * half] * inv, o[4 * (4 * g + k) + 2 * half + 1] * inv);
        attw_quad_transpose(a, c, q);
        if (row < T)
          *reinterpret_cast<uint4*>(ob + (int64_t)row * w + 8 * (4 * g + q)) =
              row < L ? make_uint4(c[0], c[1], c[2], c[3]) : make_uint4(0u, 0u, 0u, 0u);
      }
    }
  }
  // rows of the warps past the sample's keys (none without lengths): 8 x 16-byte stores per row of the head
  for (int i = 16 * ((L + 15) / 16) * 8 + (int)threadIdx.x; i < T * 8; i += ATTW_THREADS)
    *reinterpret_cast<uint4*>(ob + (int64_t)(i >> 3) * w + 8 * (i & 7)) = make_uint4(0u, 0u, 0u, 0u);
}

bool attention_wgmma_supported(int T, int heads, int w) {
  return heads > 0 && w == heads * ATTW_HD && T >= 1 && T <= ATTW_MAX_T;
}

int attention_wgmma(const CUtensorMap& tmQKV, __nv_bfloat16* out, int B, int T, int heads, int w, int causal,
                    cudaStream_t st, const int* len) {
  B200_CHECK(attention_wgmma_supported(T, heads, w), B200_ERR_UNSUPPORTED,
             "attention_wgmma: head dim 64 and T <= %d only (T=%d heads=%d w=%d)", ATTW_MAX_T, T, heads, w);
  if (B == 0) return B200_OK;
  static std::atomic<unsigned long long> configured{0};  // bit per device: the attribute is per context
  int dev = 0;
  B200_CUDA(cudaGetDevice(&dev));
  if (!(configured.load() >> (dev & 63) & 1ull)) {
    B200_CUDA(cudaFuncSetAttribute(attention_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   attw_smem_bytes(ATTW_MAX_T)));
    configured.fetch_or(1ull << (dev & 63));
  }
  const float scale_log2e = 0.125f * 1.4426950408889634f;   // hd^-0.5 * log2(e)
  attention_wgmma_kernel<<<dim3(heads, B), ATTW_THREADS, attw_smem_bytes(T), st>>>(tmQKV, out, T, w, scale_log2e, causal, len);
  B200_LAUNCH_OK();
  return B200_OK;
}

}  // namespace b200
