// OPQ training (FAISS OPQMatrix::train, restated in DESIGN §5 (xiii) and tests/opq_ref.py): a rotation A [d_out, d_in]
// with orthonormal rows that lowers the PQ error of A x.  Per iteration:
//   xproj = X A^T (pq_rows_pretransform_kernel), PQ trained on xproj (pq_train_loop, hot-started from the previous
//   codebook after the first iteration), Y = decode(codes), objective |xproj - Y|^2 / n, G = Y^T X, A = polar(G) = U V^T.
// Kernels: (1) the cross matrix G = Y^T X as 64 x 64-tile fp32 FMA over fixed 1024-row chunks, the decode fused into
// the Y operand load; each chunk writes its own partial and a second kernel adds the partials in chunk order, so G is
// the same bits on every run (no floating-point atomics); (2) the squared error per row (fp64, one warp per row);
// (3) A = U V^T from the fp64 SVD of G (cuSOLVER gesvd, resolved at run time so the library links without it).
#include "index.cuh"
#include "topk.cuh"
#include <cusolverDn.h>
#include <dlfcn.h>
#include <chrono>
#include <cmath>
#include <mutex>
#include <vector>

namespace b200 {

constexpr int OQ_KSUB = 256;
constexpr int OQ_CHUNK = 1024;        // rows per cross-matrix partial
constexpr int64_t OQ_MAX_TRAIN = 65536;   // FAISS OPQMatrix max_train_points (256 * 256)

// ---- (1) cross matrix ---------------------------------------------------------------------------------------------
// Grid (d_in / 64, d_out / 64, chunks); thread (ty, tx) owns G[i0 + ty + 16u][j0 + tx + 16v], u, v < 4, and adds the
// chunk's rows in ascending order, one fma each: P[c][i][j] = sum_r Y[r][i] X[r][j].
constexpr int CX_T = 64, CX_K = 16;
__global__ void __launch_bounds__(256)
opq_cross_kernel(const float* __restrict__ X, int64_t n, int d_in, const uint8_t* __restrict__ codes,
                 const float* __restrict__ cb, int d_out, int M, float* __restrict__ P) {
  __shared__ float sy[CX_K][CX_T + 1], sx[CX_K][CX_T + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int j0 = blockIdx.x * CX_T, i0 = blockIdx.y * CX_T;
  const int64_t rbeg = (int64_t)blockIdx.z * OQ_CHUNK;
  const int64_t rend = rbeg + OQ_CHUNK < n ? rbeg + OQ_CHUNK : n;
  const int dsub = d_out / M;
  float acc[4][4] = {};
  for (int64_t k0 = rbeg; k0 < rend; k0 += CX_K) {
    for (int e = threadIdx.x; e < CX_T * CX_K; e += 256) {
      const int rr = e / CX_T, c = e % CX_T;
      const int64_t r = k0 + rr;
      const bool live = r < rend;
      const int i = i0 + c, j = j0 + c;
      float y = 0.f;
      if (live && i < d_out) {
        const int m = i / dsub;
        y = cb[((int64_t)m * OQ_KSUB + codes[r * M + m]) * dsub + (i - m * dsub)];
      }
      sy[rr][c] = y;
      sx[rr][c] = (live && j < d_in) ? X[r * d_in + j] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int c = 0; c < CX_K; c++) {
      float a[4], b[4];
#pragma unroll
      for (int u = 0; u < 4; u++) { a[u] = sy[c][ty + 16 * u]; b[u] = sx[c][tx + 16 * u]; }
#pragma unroll
      for (int u = 0; u < 4; u++)
#pragma unroll
        for (int v = 0; v < 4; v++) acc[u][v] = fmaf(a[u], b[v], acc[u][v]);
    }
    __syncthreads();
  }
  float* out = P + (int64_t)blockIdx.z * d_out * d_in;
#pragma unroll
  for (int u = 0; u < 4; u++)
#pragma unroll
    for (int v = 0; v < 4; v++) {
      const int i = i0 + ty + 16 * u, j = j0 + tx + 16 * v;
      if (i < d_out && j < d_in) out[(int64_t)i * d_in + j] = acc[u][v];
    }
}

// G[e] = ((P[0][e] + P[1][e]) + P[2][e]) + ...: the chunk partials in chunk order.
__global__ void opq_reduce_kernel(const float* __restrict__ P, int chunks, int64_t count, float* __restrict__ G) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= count) return;
  float s = P[e];
  for (int c = 1; c < chunks; c++) s = __fadd_rn(s, P[(int64_t)c * count + e]);
  G[e] = s;
}

// ---- (2) squared reconstruction error per row: err[r] = sum_i (xproj[r][i] - Y[r][i])^2 in fp64 ------------------
__global__ void opq_error_kernel(const float* __restrict__ Xp, int64_t n, int d, const uint8_t* __restrict__ codes,
                                 const float* __restrict__ cb, int M, double* __restrict__ err) {
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  const int dsub = d / M;
  double s = 0.0;
  for (int i = lane; i < d; i += 32) {
    const int m = i / dsub;
    const double e = (double)Xp[r * d + i] - (double)cb[((int64_t)m * OQ_KSUB + codes[r * M + m]) * dsub + (i - m * dsub)];
    s += e * e;
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(FULL, s, o);
  if (lane == 0) err[r] = s;
}

// ---- (3) polar factor -----------------------------------------------------------------------------------------------
__global__ void opq_widen_kernel(const float* __restrict__ a, int64_t count, double* __restrict__ b) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < count) b[e] = (double)a[e];
}

// A[i][j] = sum_k V'[i][k] U'[j][k] in fp64, stored fp32.  gesvd of the column-major d_in x d_out matrix G^T gives
// G^T = U' S V'^T: U' column-major [d_in, d_out] (ldu d_in), V'^T column-major [d_out, d_out], so G = V' S U'^T and its
// polar factor U V^T is V' U'^T.
__global__ void opq_polar_product_kernel(const double* __restrict__ U, const double* __restrict__ VT, int d_out, int d_in,
                                         float* __restrict__ A) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y;
  if (j >= d_in) return;
  double s = 0.0;
  for (int k = 0; k < d_out; k++) s = fma(VT[k + (int64_t)i * d_out], U[j + (int64_t)k * d_in], s);
  A[(int64_t)i * d_in + j] = (float)s;
}

struct CusolverApi {
  decltype(&cusolverDnCreate) Create = nullptr;
  decltype(&cusolverDnDestroy) Destroy = nullptr;
  decltype(&cusolverDnSetStream) SetStream = nullptr;
  decltype(&cusolverDnDgesvd_bufferSize) BufferSize = nullptr;
  decltype(&cusolverDnDgesvd) Gesvd = nullptr;
  bool ok = false;
};

static const CusolverApi& cusolver() {
  static CusolverApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    void* h = dlopen("libcusolver.so.11", RTLD_NOW | RTLD_NOLOAD);   // the copy already in the process (e.g. torch's)
    if (!h) h = dlopen("libcusolver.so.11", RTLD_NOW);
    if (!h) return;
    api.Create = (decltype(api.Create))dlsym(h, "cusolverDnCreate");
    api.Destroy = (decltype(api.Destroy))dlsym(h, "cusolverDnDestroy");
    api.SetStream = (decltype(api.SetStream))dlsym(h, "cusolverDnSetStream");
    api.BufferSize = (decltype(api.BufferSize))dlsym(h, "cusolverDnDgesvd_bufferSize");
    api.Gesvd = (decltype(api.Gesvd))dlsym(h, "cusolverDnDgesvd");
    api.ok = api.Create && api.Destroy && api.SetStream && api.BufferSize && api.Gesvd;
  });
  return api;
}

// A [d_out, d_in] fp32 = the orthogonal polar factor of Gd [d_out, d_in] fp64 (overwritten), through its fp64 SVD.
static int polar_fp64(double* Gd, int d_out, int d_in, float* A, cudaStream_t st) {
  const CusolverApi& api = cusolver();
  B200_CHECK(api.ok, B200_ERR_UNSUPPORTED,
             "opq: libcusolver.so.11 (cuSOLVER, the SVD of the Procrustes step) could not be loaded");
  cusolverDnHandle_t h = nullptr;
  B200_CHECK(api.Create(&h) == CUSOLVER_STATUS_SUCCESS, B200_ERR_CUDA, "opq: cusolverDnCreate failed");
  double *S = nullptr, *U = nullptr, *VT = nullptr, *work = nullptr;
  int* info = nullptr;
  int rc = [&]() -> int {
    B200_CHECK(api.SetStream(h, st) == CUSOLVER_STATUS_SUCCESS, B200_ERR_CUDA, "opq: cusolverDnSetStream failed");
    int lwork = 0;
    B200_CHECK(api.BufferSize(h, d_in, d_out, &lwork) == CUSOLVER_STATUS_SUCCESS, B200_ERR_CUDA,
               "opq: cusolverDnDgesvd_bufferSize failed");
    B200_CUDA(cudaMalloc((void**)&S, (size_t)d_out * 8));
    B200_CUDA(cudaMalloc((void**)&U, (size_t)d_in * d_out * 8));
    B200_CUDA(cudaMalloc((void**)&VT, (size_t)d_out * d_out * 8));
    B200_CUDA(cudaMalloc((void**)&work, (size_t)std::max(lwork, 1) * 8));
    B200_CUDA(cudaMalloc((void**)&info, 4));
    B200_CHECK(api.Gesvd(h, 'S', 'A', d_in, d_out, Gd, d_in, S, U, d_in, VT, d_out, work, lwork, nullptr, info) ==
                   CUSOLVER_STATUS_SUCCESS, B200_ERR_CUDA, "opq: cusolverDnDgesvd failed");
    count_launch();
    int h_info = 0;
    B200_CUDA(cudaMemcpyAsync(&h_info, info, 4, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    B200_CHECK(h_info == 0, B200_ERR_CUDA, "opq: gesvd did not converge (info %d)", h_info);
    opq_polar_product_kernel<<<dim3((d_in + 127) / 128, d_out), 128, 0, st>>>(U, VT, d_out, d_in, A);
    B200_LAUNCH_OK();
    B200_CUDA(cudaStreamSynchronize(st));
    return B200_OK;
  }();
  api.Destroy(h);
  for (void* p : {(void*)S, (void*)U, (void*)VT, (void*)work, (void*)info}) if (p) cudaFree(p);
  return rc;
}

static int polar_f32(const float* G, int d_out, int d_in, float* A, cudaStream_t st) {
  const int64_t count = (int64_t)d_out * d_in;
  double* Gd = nullptr;
  B200_CUDA(cudaMalloc((void**)&Gd, (size_t)count * 8));
  int rc = [&]() -> int {
    opq_widen_kernel<<<(unsigned)((count + 255) / 256), 256, 0, st>>>(G, count, Gd);
    B200_LAUNCH_OK();
    return polar_fp64(Gd, d_out, d_in, A, st);
  }();
  cudaStreamSynchronize(st);
  cudaFree(Gd);
  return rc;
}

static int cross(const float* X, int64_t n, int d_in, const uint8_t* codes, const float* cb, int d_out, int M, float* P,
                 float* G, cudaStream_t st) {
  const int chunks = (int)((n + OQ_CHUNK - 1) / OQ_CHUNK);
  const int64_t count = (int64_t)d_out * d_in;
  opq_cross_kernel<<<dim3((d_in + CX_T - 1) / CX_T, (d_out + CX_T - 1) / CX_T, chunks), 256, 0, st>>>(X, n, d_in, codes, cb,
                                                                                                     d_out, M, P);
  B200_LAUNCH_OK();
  opq_reduce_kernel<<<(unsigned)((count + 255) / 256), 256, 0, st>>>(P, chunks, count, G);
  B200_LAUNCH_OK();
  return B200_OK;
}

static uint64_t opq_mix(uint64_t x) {   // pq_mix / kmeans_mix: splitmix64's finaliser
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

// Entry e of the seeded Gaussian matrix: Box-Muller on two counter-based uniforms,
// u1 = (h(2e) >> 11 + 1) 2^-53 in (0, 1], u2 = (h(2e + 1) >> 11) 2^-53, h(c) = mix(seed ^ c * 0xD1342543DE82EF95).
static double opq_gaussian(uint64_t seed, uint64_t e) {
  const uint64_t a = opq_mix(seed ^ ((2 * e) * 0xD1342543DE82EF95ull));
  const uint64_t b = opq_mix(seed ^ ((2 * e + 1) * 0xD1342543DE82EF95ull));
  const double u1 = (double)((a >> 11) + 1) * 0x1p-53, u2 = (double)(b >> 11) * 0x1p-53;
  return std::sqrt(-2.0 * std::log(u1)) * std::cos(6.283185307179586 * u2);
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_opq_cross_f32_device(const float* d_x, int64_t n, int d_in, const uint8_t* d_codes, const float* d_codebook,
                              int d_out, int M, float* d_G, int device, void* stream) {
  B200_CHECK(d_x && d_codes && d_codebook && d_G && n >= 1, B200_ERR_INVALID, "opq_cross: bad argument");
  B200_CHECK(n <= OQ_MAX_TRAIN, B200_ERR_INVALID, "opq_cross: n=%lld rows; at most 65536 (the OPQ training sample)",
             (long long)n);
  B200_CHECK(d_in >= 1 && d_out >= 1 && M >= 1 && d_out % M == 0, B200_ERR_INVALID,
             "opq_cross: M=%d must divide d_out=%d (d_in=%d)", M, d_out, d_in);
  DeviceGuard g(device);
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t chunks = (n + OQ_CHUNK - 1) / OQ_CHUNK;
  float* P = nullptr;
  B200_CUDA(cudaMallocAsync((void**)&P, (size_t)chunks * d_out * d_in * 4, st));
  const int rc = cross(d_x, n, d_in, d_codes, d_codebook, d_out, M, P, d_G, st);
  const cudaError_t e = cudaFreeAsync(P, st);
  if (rc == B200_OK) B200_CUDA(e);
  return rc;
}

int b200_opq_polar_f32_device(const float* d_G, int d_out, int d_in, float* d_A, int device, void* stream) {
  B200_CHECK(d_G && d_A && d_out >= 1 && d_out <= d_in, B200_ERR_INVALID,
             "opq_polar: bad argument (d_out=%d must be in [1, d_in=%d])", d_out, d_in);
  DeviceGuard g(device);
  return polar_f32(d_G, d_out, d_in, d_A, (cudaStream_t)stream);
}

int b200_opq_train_f32(const float* d_x, int64_t n, int d_in, int d_out, int M, int niter, int niter_pq, int niter_pq_0,
                       uint64_t seed, float* h_A, float* h_objective, float* h_phase_ms, int device) {
  B200_CHECK(d_x && h_A, B200_ERR_INVALID, "opq_train: null argument");
  B200_CHECK(d_out >= 1 && d_out <= d_in, B200_ERR_INVALID, "opq_train: d_out=%d must be in [1, d_in=%d]", d_out, d_in);
  B200_CHECK(M >= 1 && d_out % M == 0, B200_ERR_INVALID, "opq_train: M=%d must divide d_out=%d", M, d_out);
  B200_CHECK(n >= OQ_KSUB && n <= OQ_MAX_TRAIN, B200_ERR_INVALID,
             "opq_train: n=%lld training rows must be in [256, 65536] (pick a sample first)", (long long)n);
  B200_CHECK(niter >= 0 && niter_pq >= 0 && niter_pq_0 >= 0, B200_ERR_INVALID, "opq_train: negative iteration count");
  DeviceGuard g(device);
  const int64_t count = (int64_t)d_out * d_in, chunks = (n + OQ_CHUNK - 1) / OQ_CHUNK;
  float *A = nullptr, *xp = nullptr, *cb = nullptr, *P = nullptr, *G = nullptr;
  double *Gd = nullptr, *err = nullptr;
  uint8_t* codes = nullptr;
  std::vector<void*> frees;
  auto alloc = [&](void** p, size_t bytes) -> int {
    B200_CUDA(cudaMalloc(p, bytes));
    frees.push_back(*p);
    return B200_OK;
  };
  int rc = [&]() -> int {
    B200_TRY(alloc((void**)&A, (size_t)count * 4));
    B200_TRY(alloc((void**)&Gd, (size_t)count * 8));
    B200_TRY(alloc((void**)&xp, (size_t)n * d_out * 4));
    B200_TRY(alloc((void**)&cb, (size_t)OQ_KSUB * d_out * 4));
    B200_TRY(alloc((void**)&codes, (size_t)n * M));
    B200_TRY(alloc((void**)&P, (size_t)chunks * count * 4));
    B200_TRY(alloc((void**)&G, (size_t)count * 4));
    B200_TRY(alloc((void**)&err, (size_t)n * 8));
    // phase timing (h_phase_ms): wall time between device synchronisations, added per phase
    double phase[4] = {0, 0, 0, 0};
    auto t_last = std::chrono::steady_clock::now();
    auto mark = [&](int ph) -> int {
      if (!h_phase_ms) return B200_OK;
      B200_CUDA(cudaDeviceSynchronize());
      const auto t = std::chrono::steady_clock::now();
      phase[ph] += std::chrono::duration<double, std::milli>(t - t_last).count();
      t_last = t;
      return B200_OK;
    };
    // initial rotation: the polar factor of a seeded Gaussian d_out x d_in matrix
    std::vector<double> gauss((size_t)count);
    for (int64_t e = 0; e < count; e++) gauss[e] = opq_gaussian(seed, (uint64_t)e);
    B200_CUDA(cudaMemcpy(Gd, gauss.data(), (size_t)count * 8, cudaMemcpyHostToDevice));
    B200_TRY(polar_fp64(Gd, d_out, d_in, A, 0));
    B200_TRY(mark(3));
    std::vector<double> h_err((size_t)n);
    for (int it = 0; it < niter; it++) {
      B200_TRY(pq_pretransform(d_x, n, d_in, A, nullptr, d_out, xp, 0));
      B200_TRY(mark(0));
      if (it == 0) B200_TRY(pq_init_codebook(xp, n, d_out, M, seed, cb));
      B200_TRY(pq_train_loop(xp, n, d_out, M, it == 0 ? niter_pq_0 : niter_pq, cb, codes, nullptr));
      opq_error_kernel<<<(unsigned)((n + 7) / 8), 256>>>(xp, n, d_out, codes, cb, M, err);
      B200_LAUNCH_OK();
      B200_CUDA(cudaMemcpy(h_err.data(), err, (size_t)n * 8, cudaMemcpyDeviceToHost));
      if (h_objective) {
        double s = 0.0;
        for (int64_t r = 0; r < n; r++) s += h_err[r];
        h_objective[it] = (float)(s / (double)n);
      }
      B200_TRY(mark(1));
      B200_TRY(cross(d_x, n, d_in, codes, cb, d_out, M, P, G, 0));
      B200_TRY(mark(2));
      opq_widen_kernel<<<(unsigned)((count + 255) / 256), 256>>>(G, count, Gd);
      B200_LAUNCH_OK();
      B200_TRY(polar_fp64(Gd, d_out, d_in, A, 0));
      B200_TRY(mark(3));
    }
    if (h_phase_ms)
      for (int i = 0; i < 4; i++) h_phase_ms[i] = (float)phase[i];
    B200_CUDA(cudaMemcpy(h_A, A, (size_t)count * 4, cudaMemcpyDeviceToHost));
    return B200_OK;
  }();
  cudaDeviceSynchronize();
  for (void* p : frees) cudaFree(p);
  return rc;
}

}  // extern "C"
