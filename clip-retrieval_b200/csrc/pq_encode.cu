// IVF-PQ encoding and PQ training (8-bit codes, inner-product coarse quantiser): the writer side of knn_ivfpq.cu.
// FAISS IndexIVFPQ semantics, as restated in DESIGN §5 (ix) and tests/pq_train_ref.py:
//   x' = A x + b (when a pre-transform is set), else x;
//   list(x) = argmax_l x' . c_l over the fp32 centroids, ties to the lower list id (the rule of the search's coarse step);
//   r = x' - c_list in fp32 when by_residual, else x';
//   code_m = argmin_j sum_t (r[m dsub + t] - cb[m][j][t])^2 in fp32, ties to the lower j.  The direct difference form is
//   used on purpose instead of FAISS's |r|^2 + |c|^2 - 2 r.c, which cancels for residuals close to a codeword.
// Kernels: (1) the row pre-transform as a 64 x 64-tile fp32 GEMM; (2) the fused coarse assignment: a 128 x 128-tile
// fp32 FMA GEMM of rows x centroids whose CTA keeps a running argmax over every list tile and writes one int32 per
// row (no score matrix: at 65 536 rows x 65 536 lists it would take 34 GB); (3) codeword assignment with the residual
// taken on load, the codebook of one sub-quantiser staged in shared memory in column chunks; (4) the PQ k-means update
// (stable radix sort by (m, code), one CTA per (m, j) adding its rows in ascending row order, then the splits of
// empty clusters).
#include "index.cuh"
#include "topk.cuh"
#include <cub/cub.cuh>
#include <algorithm>
#include <mutex>
#include <vector>

namespace b200 {

constexpr int PE_KSUB = 256;
constexpr int64_t PE_CHUNK = 32768;   // rows per encode chunk: bounds the scratch (pre-transformed rows, lists)

// ---- (1) row pre-transform: Y[n, d] = X[n, d_in] A^T (+ b), 64 x 64 tiles, 4 x 4 per thread ---------------------
constexpr int PT_T = 64, PT_K = 16;
template <typename OutT>   // float (encode) or __half (training rows a caller keeps in fp16)
__global__ void __launch_bounds__(256)
pq_rows_pretransform_kernel(const float* __restrict__ X, int64_t n, int d_in, const float* __restrict__ A,
                            const float* __restrict__ b, int d, OutT* __restrict__ Y) {
  __shared__ float sx[PT_K][PT_T + 1], sa[PT_K][PT_T + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int i0 = blockIdx.x * PT_T;
  const int64_t r0 = (int64_t)blockIdx.y * PT_T;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < d_in; k0 += PT_K) {
    for (int i = threadIdx.x; i < PT_T * PT_K; i += 256) {
      const int r = i / PT_K, c = i % PT_K;
      sx[c][r] = (r0 + r < n && k0 + c < d_in) ? X[(r0 + r) * d_in + k0 + c] : 0.f;
      sa[c][r] = (i0 + r < d && k0 + c < d_in) ? A[(int64_t)(i0 + r) * d_in + k0 + c] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int c = 0; c < PT_K; c++) {
      float a[4], bb[4];
#pragma unroll
      for (int u = 0; u < 4; u++) { a[u] = sx[c][ty + 16 * u]; bb[u] = sa[c][tx + 16 * u]; }
#pragma unroll
      for (int u = 0; u < 4; u++)
#pragma unroll
        for (int v = 0; v < 4; v++) acc[u][v] = fmaf(a[u], bb[v], acc[u][v]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int u = 0; u < 4; u++)
#pragma unroll
    for (int v = 0; v < 4; v++) {
      const int64_t r = r0 + ty + 16 * u;
      const int i = i0 + tx + 16 * v;
      if (r < n && i < d) Y[r * d + i] = (OutT)(b ? acc[u][v] + b[i] : acc[u][v]);
    }
}

// ---- (2) fused coarse assignment ---------------------------------------------------------------------------------
// One CTA per 128 rows loops over all lists in tiles of 128; thread (ty, tx) accumulates rows {4ty..4ty+3, 64+4ty..}
// x lists {4tx..4tx+3, 64+4tx..} over d in chunks of 8 (float4 shared-memory reads: 4 loads per 64 FMAs; the next
// chunk's global loads are issued before the current chunk's FMAs).  Each score becomes a key (ordered score, ~list):
// the larger key is the higher score, then the lower list id, so one unsigned max per (row, list) keeps the running
// argmax inside a tile and across tiles, and a shuffle max over the 16 threads of a row finishes it.  NaN scores are
// never kept; a row whose every score is NaN gets list 0.  Needs d % 8 == 0 and 16-byte aligned rows.
constexpr int AS_BM = 128, AS_BN = 128, AS_BK = 8;
__global__ void __launch_bounds__(256)
pq_assign_kernel(const float* __restrict__ X, int64_t n, const float* __restrict__ Cn, int nlist, int d,
                 int32_t* __restrict__ lists) {
  __shared__ __align__(16) float sx[AS_BK][AS_BM];
  __shared__ __align__(16) float sc[AS_BK][AS_BN];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t r0 = (int64_t)blockIdx.x * AS_BM;
  const int lr = tid >> 1, lc = (tid & 1) * 4;   // loader: row / list lr, columns lc..lc+3 of the chunk
  const bool xlive = r0 + lr < n;
  const float* xrow = X + (xlive ? r0 + lr : 0) * (int64_t)d + lc;
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  unsigned long long best[8];
#pragma unroll
  for (int u = 0; u < 8; u++) best[u] = 0ull;
  for (int l0 = 0; l0 < nlist; l0 += AS_BN) {
    const bool clive = l0 + lr < nlist;
    const float* crow = Cn + (int64_t)(clive ? l0 + lr : 0) * d + lc;
    float acc[8][8];
#pragma unroll
    for (int u = 0; u < 8; u++)
#pragma unroll
      for (int v = 0; v < 8; v++) acc[u][v] = 0.f;
    float4 xv = xlive ? __ldg(reinterpret_cast<const float4*>(xrow)) : zero;
    float4 cv = clive ? __ldg(reinterpret_cast<const float4*>(crow)) : zero;
    for (int k0 = 0; k0 < d; k0 += AS_BK) {
      __syncthreads();   // the previous chunk has been read
      sx[lc + 0][lr] = xv.x; sx[lc + 1][lr] = xv.y; sx[lc + 2][lr] = xv.z; sx[lc + 3][lr] = xv.w;
      sc[lc + 0][lr] = cv.x; sc[lc + 1][lr] = cv.y; sc[lc + 2][lr] = cv.z; sc[lc + 3][lr] = cv.w;
      __syncthreads();
      if (k0 + AS_BK < d) {
        xv = xlive ? __ldg(reinterpret_cast<const float4*>(xrow + k0 + AS_BK)) : zero;
        cv = clive ? __ldg(reinterpret_cast<const float4*>(crow + k0 + AS_BK)) : zero;
      }
#pragma unroll
      for (int c = 0; c < AS_BK; c++) {
        const float4 a0 = *reinterpret_cast<const float4*>(&sx[c][ty * 4]);
        const float4 a1 = *reinterpret_cast<const float4*>(&sx[c][64 + ty * 4]);
        const float4 b0 = *reinterpret_cast<const float4*>(&sc[c][tx * 4]);
        const float4 b1 = *reinterpret_cast<const float4*>(&sc[c][64 + tx * 4]);
        const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int u = 0; u < 8; u++)
#pragma unroll
          for (int v = 0; v < 8; v++) acc[u][v] = fmaf(a[u], bb[v], acc[u][v]);
      }
    }
#pragma unroll
    for (int v = 0; v < 8; v++) {
      const int l = l0 + (v < 4 ? tx * 4 + v : 64 + tx * 4 + v - 4);
      if (l < nlist)
#pragma unroll
        for (int u = 0; u < 8; u++) {
          const unsigned long long key = make_key(acc[u][v], (uint32_t)l);
          if (acc[u][v] == acc[u][v] && key > best[u]) best[u] = key;
        }
    }
  }
#pragma unroll
  for (int u = 0; u < 8; u++) {
#pragma unroll
    for (int o = 8; o >= 1; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(FULL, best[u], o);
      if (other > best[u]) best[u] = other;
    }
    const int64_t row = r0 + (u < 4 ? ty * 4 + u : 64 + ty * 4 + u - 4);
    if (tx == 0 && row < n) lists[row] = best[u] ? (int32_t)key_id(best[u]) : 0;
  }
}

// ---- (3) codeword assignment -------------------------------------------------------------------------------------
// Grid (row blocks of CW_ROWS, M).  Thread j scores codeword j of sub-quantiser m against CW_R rows per pass.  Column
// chunks of at most CW_TC: the codebook chunk sits transposed in shared memory ([t][j], conflict-free), the residual
// chunk of the pass's rows beside it (r = x' - c_list on load, written to `res_out` when asked); when one chunk
// covers dsub the codebook is loaded once per CTA.  Each distance is a sequential fp32 sum over t of (r_t - cb_t)^2
// (one rounded subtraction, one fma).  Argmin over j: min of (distance bits << 32 | j) (distances are >= +0, so their
// bits order as the values; NaN never wins), ties to the lower j.
constexpr int CW_R = 16, CW_TC = 32, CW_ROWS = 256;
__global__ void __launch_bounds__(256)
pq_code_kernel(const float* __restrict__ X, int64_t n, int d, int M, int dsub, const float* __restrict__ cb,
               const float* __restrict__ cent, const int32_t* __restrict__ lists, float* __restrict__ res_out,
               uint8_t* __restrict__ codes) {
  __shared__ float s_cb[CW_TC][PE_KSUB];
  __shared__ float s_r[CW_R][CW_TC];
  __shared__ unsigned long long s_red[8][CW_R];
  const int j = threadIdx.x, lane = j & 31, warp = j >> 5;
  const int m = blockIdx.y;
  const int64_t rbeg = (int64_t)blockIdx.x * CW_ROWS;
  const int64_t rend = rbeg + CW_ROWS < n ? rbeg + CW_ROWS : n;
  const float* cbm = cb + (int64_t)m * PE_KSUB * dsub;
  const int nch = (dsub + CW_TC - 1) / CW_TC;
  for (int64_t p0 = rbeg; p0 < rend; p0 += CW_R) {
    float acc[CW_R];
#pragma unroll
    for (int rr = 0; rr < CW_R; rr++) acc[rr] = 0.f;
    for (int ch = 0; ch < nch; ch++) {
      const int t0 = ch * CW_TC, tw = min(CW_TC, dsub - t0);
      __syncthreads();
      if (nch > 1 || p0 == rbeg)
        for (int i = j; i < PE_KSUB * tw; i += blockDim.x) {
          const int jj = i / tw, t = i - jj * tw;
          s_cb[t][jj] = cbm[(int64_t)jj * dsub + t0 + t];
        }
      for (int i = j; i < CW_R * tw; i += blockDim.x) {
        const int rr = i / tw, t = i - rr * tw;
        const int64_t row = p0 + rr;
        float v = 0.f;
        if (row < rend) {
          const int col = m * dsub + t0 + t;
          v = X[row * d + col];
          if (cent) v = __fsub_rn(v, cent[(int64_t)lists[row] * d + col]);
          if (res_out) res_out[row * d + col] = v;
        }
        s_r[rr][t] = v;
      }
      __syncthreads();
      for (int t = 0; t < tw; t++) {
        const float c = s_cb[t][j];
#pragma unroll
        for (int rr = 0; rr < CW_R; rr++) {
          const float e = __fsub_rn(s_r[rr][t], c);
          acc[rr] = fmaf(e, e, acc[rr]);
        }
      }
    }
    if (!codes) continue;
#pragma unroll
    for (int rr = 0; rr < CW_R; rr++) {
      unsigned long long key = acc[rr] == acc[rr] ? ((unsigned long long)__float_as_uint(acc[rr]) << 32) | (uint32_t)j : ~0ull;
#pragma unroll
      for (int o = 16; o >= 1; o >>= 1) {
        const unsigned long long other = __shfl_xor_sync(FULL, key, o);
        if (other < key) key = other;
      }
      if (lane == 0) s_red[warp][rr] = key;
    }
    __syncthreads();
    if (j < CW_R && p0 + j < rend) {
      unsigned long long key = s_red[0][j];
      for (int w = 1; w < (int)(blockDim.x >> 5); w++) key = s_red[w][j] < key ? s_red[w][j] : key;
      codes[(p0 + j) * M + m] = key == ~0ull ? 0 : (uint8_t)(key & 0xffu);
    }
  }
}

// ---- (4) PQ k-means ----------------------------------------------------------------------------------------------
// Initial codewords: cb[m][j] = sub-vector m of row pick[j] (the same picks for every m).
__global__ void pq_gather_kernel(const float* __restrict__ X, int d, int dsub, const int64_t* __restrict__ pick,
                                 float* __restrict__ cb) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;   // over [M, 256, dsub]
  if (i >= (int64_t)PE_KSUB * d) return;
  const int t = (int)(i % dsub);
  const int64_t mj = i / dsub;
  const int jj = (int)(mj % PE_KSUB), m = (int)(mj / PE_KSUB);
  cb[i] = X[pick[jj] * d + (int64_t)m * dsub + t];
}

// Sort keys m * 256 + code_m of every (m, row), stored m-major so that a stable sort leaves each (m, j) bucket in
// ascending row order; values = row.
__global__ void pq_sort_keys_kernel(const uint8_t* __restrict__ codes, int64_t n, int M, uint32_t* __restrict__ keys,
                                    uint32_t* __restrict__ rows) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;   // over [M, n]
  if (i >= (int64_t)M * n) return;
  const int m = (int)(i / n);
  const int64_t r = i - (int64_t)m * n;
  keys[i] = (uint32_t)m * PE_KSUB + codes[r * M + m];
  rows[i] = (uint32_t)r;
}

// off[b] = first position of sorted `keys` holding a key >= b, b in [0, nb].
__global__ void pq_offsets_kernel(const uint32_t* __restrict__ keys, int64_t count, int nb, int64_t* __restrict__ off) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b > nb) return;
  int64_t lo = 0, hi = count;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (keys[mid] < (uint32_t)b) lo = mid + 1; else hi = mid;
  }
  off[b] = lo;
}

// One CTA per (m, j): codeword = (sum of its rows' sub-vectors, added in ascending row order in fp32) * (1 / count).
// An empty bucket keeps its codeword until the split step.
__global__ void pq_update_kernel(const float* __restrict__ R, int d, int dsub, const uint32_t* __restrict__ sorted_rows,
                                 const int64_t* __restrict__ off, float* __restrict__ cb) {
  const int bkt = blockIdx.x, m = bkt / PE_KSUB;
  const int64_t p0 = off[bkt], p1 = off[bkt + 1];
  if (p1 == p0) return;
  const float inv = 1.0f / (float)(p1 - p0);
  for (int t = threadIdx.x; t < dsub; t += blockDim.x) {
    float s = 0.f;
    for (int64_t p = p0; p < p1; p++) s = __fadd_rn(s, R[(int64_t)sorted_rows[p] * d + (int64_t)m * dsub + t]);
    cb[(int64_t)bkt * dsub + t] = s * inv;
  }
}

// kmeans_split_kernel (knn_ivf.cu) on dsub-strided codewords, for a list of (m, ci, cj) applied in order: the empty
// codeword ci of sub-quantiser m takes codeword cj, the two perturbed by 1 +- 1/1024, alternating by column.
__global__ void pq_split_kernel(float* __restrict__ cb, int dsub, const int* __restrict__ splits, int count) {
  const float eps = 1.0f / 1024.0f;
  for (int s = 0; s < count; s++) {
    const int m = splits[3 * s], ci = splits[3 * s + 1], cj = splits[3 * s + 2];
    float* a = cb + ((int64_t)m * PE_KSUB + ci) * dsub;
    float* b = cb + ((int64_t)m * PE_KSUB + cj) * dsub;
    for (int t = threadIdx.x; t < dsub; t += blockDim.x) {
      const float v = b[t];
      a[t] = (t % 2 == 0) ? v * (1.0f + eps) : v * (1.0f - eps);
      b[t] = (t % 2 == 0) ? v * (1.0f - eps) : v * (1.0f + eps);
    }
    __syncthreads();
  }
}

static inline uint64_t pq_mix(uint64_t x) {   // kmeans_mix (knn_ivf.cu): the same seeded picks
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

static int launch_code(const float* X, int64_t n, int d, int M, const float* cb, const float* cent, const int32_t* lists,
                       float* res_out, uint8_t* codes, cudaStream_t st) {
  if (n == 0) return B200_OK;
  pq_code_kernel<<<dim3((unsigned)((n + CW_ROWS - 1) / CW_ROWS), (unsigned)M), 256, 0, st>>>(X, n, d, M, d / M, cb, cent,
                                                                                              lists, res_out, codes);
  B200_LAUNCH_OK();
  return B200_OK;
}

int pq_codes(const float* X, int64_t n, int d, int M, const float* cb, uint8_t* codes, cudaStream_t st) {
  return launch_code(X, n, d, M, cb, nullptr, nullptr, nullptr, codes, st);
}

int pq_pretransform(const float* X, int64_t n, int d_in, const float* A, const float* b, int d, float* Y, cudaStream_t st) {
  if (n == 0) return B200_OK;
  pq_rows_pretransform_kernel<float><<<dim3((d + PT_T - 1) / PT_T, (unsigned)((n + PT_T - 1) / PT_T)), 256, 0, st>>>(
      X, n, d_in, A, b, d, Y);
  B200_LAUNCH_OK();
  return B200_OK;
}

int pq_init_codebook(const float* d_x, int64_t n, int d, int M, uint64_t seed, float* cb) {
  // one seeded pick inside each of 256 equal strides of the rows (oracle/kmeans_ref.initial_picks)
  std::vector<int64_t> pick(PE_KSUB);
  for (int i = 0; i < PE_KSUB; i++) {
    const int64_t lo = (int64_t)(((__int128)i * n) / PE_KSUB), hi = (int64_t)(((__int128)(i + 1) * n) / PE_KSUB);
    const uint64_t span = (uint64_t)std::max<int64_t>(1, hi - lo);
    pick[i] = lo + (int64_t)(pq_mix(seed ^ ((uint64_t)i * 0xD1342543DE82EF95ull)) % span);
  }
  int64_t* d_pick = nullptr;
  B200_CUDA(cudaMalloc((void**)&d_pick, PE_KSUB * 8));
  int rc = [&]() -> int {
    B200_CUDA(cudaMemcpy(d_pick, pick.data(), PE_KSUB * 8, cudaMemcpyHostToDevice));
    pq_gather_kernel<<<(unsigned)(((int64_t)PE_KSUB * d + 255) / 256), 256>>>(d_x, d, d / M, d_pick, cb);
    B200_LAUNCH_OK();
    return B200_OK;
  }();
  cudaDeviceSynchronize();
  cudaFree(d_pick);
  return rc;
}

int pq_train_loop(const float* d_x, int64_t n, int d, int M, int niter, float* cb, uint8_t* codes_out, int64_t* h_sizes) {
  const int dsub = d / M, nb = M * PE_KSUB;
  const int64_t count = (int64_t)M * n;
  int64_t* d_off = nullptr; uint8_t* codes = codes_out;
  uint32_t *keys = nullptr, *keys2 = nullptr, *rows = nullptr, *rows2 = nullptr;
  int* d_splits = nullptr;
  void* tmp = nullptr;
  std::vector<void*> frees;
  auto alloc = [&](void** p, size_t bytes) -> int {
    B200_CUDA(cudaMalloc(p, bytes));
    frees.push_back(*p);
    return B200_OK;
  };
  int rc = [&]() -> int {
    B200_TRY(alloc((void**)&d_off, (size_t)(nb + 1) * 8));
    if (!codes) B200_TRY(alloc((void**)&codes, (size_t)count));
    B200_TRY(alloc((void**)&keys, (size_t)count * 4));
    B200_TRY(alloc((void**)&keys2, (size_t)count * 4));
    B200_TRY(alloc((void**)&rows, (size_t)count * 4));
    B200_TRY(alloc((void**)&rows2, (size_t)count * 4));
    B200_TRY(alloc((void**)&d_splits, (size_t)nb * 3 * 4));
    int bits = 1;
    while ((1ll << bits) < nb) bits++;
    size_t tmp_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys, keys2, rows, rows2, (int)count, 0, bits);
    B200_TRY(alloc(&tmp, tmp_bytes));
    const int ublock = std::min(256, (dsub + 31) / 32 * 32);
    std::vector<int64_t> off(nb + 1);
    for (int it = 0; it <= niter; it++) {
      // all M sub-quantisers in one launch per step: assign, sort by (m, code), bucket offsets
      B200_TRY(launch_code(d_x, n, d, M, cb, nullptr, nullptr, nullptr, codes, 0));
      pq_sort_keys_kernel<<<(unsigned)((count + 255) / 256), 256>>>(codes, n, M, keys, rows);
      B200_LAUNCH_OK();
      cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keys, keys2, rows, rows2, (int)count, 0, bits);
      count_launch(4);
      pq_offsets_kernel<<<(nb + 1 + 255) / 256, 256>>>(keys2, count, nb, d_off);
      B200_LAUNCH_OK();
      B200_CUDA(cudaMemcpy(off.data(), d_off, (size_t)(nb + 1) * 8, cudaMemcpyDeviceToHost));
      if (it == niter) break;   // the last round only refreshes the codes and sizes of the final codewords
      pq_update_kernel<<<nb, ublock>>>(d_x, d, dsub, rows2, d_off, cb);
      B200_LAUNCH_OK();
      // empty codewords: per m, split the (currently) largest one, ties to the lower id; sizes halve as in FAISS
      std::vector<int> splits;
      for (int m = 0; m < M; m++) {
        std::vector<int64_t> sz(PE_KSUB);
        for (int jj = 0; jj < PE_KSUB; jj++) sz[jj] = off[m * PE_KSUB + jj + 1] - off[m * PE_KSUB + jj];
        for (int ci = 0; ci < PE_KSUB; ci++) {
          if (sz[ci] != 0) continue;
          int cj = 0;
          for (int l = 1; l < PE_KSUB; l++)
            if (sz[l] > sz[cj]) cj = l;
          if (sz[cj] < 2) break;
          splits.insert(splits.end(), {m, ci, cj});
          sz[ci] = sz[cj] / 2;
          sz[cj] -= sz[ci];
        }
      }
      if (!splits.empty()) {
        B200_CUDA(cudaMemcpy(d_splits, splits.data(), splits.size() * 4, cudaMemcpyHostToDevice));
        pq_split_kernel<<<1, ublock>>>(cb, dsub, d_splits, (int)(splits.size() / 3));
        B200_LAUNCH_OK();
      }
    }
    if (h_sizes)
      for (int b = 0; b < nb; b++) h_sizes[b] = off[b + 1] - off[b];
    return B200_OK;
  }();
  cudaDeviceSynchronize();
  for (void* p : frees) cudaFree(p);
  return rc;
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_pq_train_f32(const float* d_x, int64_t n, int d, int M, int niter, uint64_t seed, float* h_codebook,
                      int64_t* h_sizes, int device) {
  B200_CHECK(d_x && h_codebook, B200_ERR_INVALID, "pq_train: null argument");
  B200_CHECK(d >= 1 && M >= 1 && M <= d && d % M == 0, B200_ERR_INVALID, "pq_train: M=%d must divide d=%d", M, d);
  B200_CHECK(n >= PE_KSUB, B200_ERR_INVALID, "pq_train: n=%lld training rows; 256 codewords need at least 256",
             (long long)n);
  B200_CHECK((int64_t)M * n < (1ll << 31) && niter >= 0, B200_ERR_INVALID,
             "pq_train: M * n = %lld must stay below 2^31 (niter=%d)", (long long)M * n, niter);
  DeviceGuard g(device);
  float* cb = nullptr;
  B200_CUDA(cudaMalloc((void**)&cb, (size_t)PE_KSUB * d * 4));
  int rc = [&]() -> int {
    B200_TRY(pq_init_codebook(d_x, n, d, M, seed, cb));
    B200_TRY(pq_train_loop(d_x, n, d, M, niter, cb, nullptr, h_sizes));
    B200_CUDA(cudaMemcpy(h_codebook, cb, (size_t)PE_KSUB * d * 4, cudaMemcpyDeviceToHost));
    return B200_OK;
  }();
  cudaDeviceSynchronize();
  cudaFree(cb);
  return rc;
}

int b200_rows_pretransform_device(const float* d_x, int64_t n, int d_in, const float* d_A, const float* d_b, int d_out,
                                  void* d_y, int out_fp16, int device, void* stream) {
  B200_CHECK(n >= 0 && (n == 0 || (d_x && d_A && d_y)) && d_in >= 1 && d_out >= 1, B200_ERR_INVALID,
             "rows_pretransform: bad argument");
  B200_CHECK(n < (1ll << 31) * PT_T, B200_ERR_INVALID, "rows_pretransform: n=%lld rows in one call", (long long)n);
  if (n == 0) return B200_OK;
  DeviceGuard g(device);
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid((d_out + PT_T - 1) / PT_T, (unsigned)((n + PT_T - 1) / PT_T));
  if (out_fp16)
    pq_rows_pretransform_kernel<__half><<<grid, 256, 0, st>>>(d_x, n, d_in, d_A, d_b, d_out, (__half*)d_y);
  else
    pq_rows_pretransform_kernel<float><<<grid, 256, 0, st>>>(d_x, n, d_in, d_A, d_b, d_out, (float*)d_y);
  B200_LAUNCH_OK();
  return B200_OK;
}

int b200_index_encode_device(b200_index* idx, const float* d_x, int64_t n, int32_t* d_lists, float* d_residuals,
                             uint8_t* d_codes, void* stream) {
  B200_CHECK(idx && n >= 0 && (d_x || n == 0), B200_ERR_INVALID, "encode: bad argument");
  B200_CHECK(idx->pq_M > 0, B200_ERR_STATE, "encode: not an IVF-PQ index");
  if (n == 0 || (!d_lists && !d_residuals && !d_codes)) return B200_OK;
  DeviceGuard g(idx->device);
  std::lock_guard<std::mutex> lock(idx->mu);
  B200_CHECK(idx->pt_A || ((uintptr_t)d_x & 15) == 0, B200_ERR_INVALID, "encode: rows must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int d = idx->d, d_in = idx->d_in, M = idx->pq_M, nlist = idx->nlist;
  const bool need_lists = d_lists || idx->pq_by_residual;   // without residuals, codes alone need no list
  const int64_t cap = std::min(n, PE_CHUNK);
  const size_t xt_bytes = idx->pt_A ? (size_t)cap * d * 4 : 0;
  const size_t l_bytes = (need_lists && !d_lists) ? (size_t)cap * 4 : 0;
  char* scratch = nullptr;
  if (xt_bytes + l_bytes) B200_CUDA(cudaMallocAsync((void**)&scratch, xt_bytes + l_bytes, st));
  int rc = [&]() -> int {
    for (int64_t r0 = 0; r0 < n; r0 += PE_CHUNK) {
      const int64_t m_ = std::min(PE_CHUNK, n - r0);
      const float* x = d_x + r0 * d_in;
      if (idx->pt_A) {
        float* xt = reinterpret_cast<float*>(scratch);
        pq_rows_pretransform_kernel<float><<<dim3((d + PT_T - 1) / PT_T, (unsigned)((m_ + PT_T - 1) / PT_T)), 256, 0, st>>>(
            x, m_, d_in, idx->pt_A, idx->pt_b, d, xt);
        B200_LAUNCH_OK();
        x = xt;
      }
      int32_t* L = d_lists ? d_lists + r0 : reinterpret_cast<int32_t*>(scratch + xt_bytes);
      if (need_lists) {
        pq_assign_kernel<<<(unsigned)((m_ + AS_BM - 1) / AS_BM), 256, 0, st>>>(x, m_, idx->pq_centroids, nlist, d, L);
        B200_LAUNCH_OK();
      }
      if (d_codes || d_residuals)
        B200_TRY(launch_code(x, m_, d, M, idx->pq_codebook, idx->pq_by_residual ? idx->pq_centroids : nullptr, L,
                             d_residuals ? d_residuals + r0 * d : nullptr, d_codes ? d_codes + r0 * M : nullptr, st));
    }
    return B200_OK;
  }();
  if (scratch) {
    const cudaError_t e = cudaFreeAsync(scratch, st);
    if (rc == B200_OK && e != cudaSuccess) B200_CUDA(e);
  }
  return rc;
}

}  // extern "C"
