// Synthetic rows for the BASELINE.json configs: counter-based, integer arithmetic up to the final
// fp64 sqrt/divide so that oracle/synth_ref.py reproduces every fp16 bit on the CPU.
#include "common.cuh"

namespace b200 {

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__host__ __device__ __forceinline__ uint64_t row_key(uint64_t seed, uint64_t row) {
  return mix64(seed ^ (row * 0x9E3779B97F4A7C15ull));
}
__host__ __device__ __forceinline__ int noise_at(uint64_t rkey, uint32_t col) {
  uint64_t h = mix64(rkey + (uint64_t)col * 0xD1342543DE82EF95ull);
  return (int)(h & 0xFF) + (int)((h >> 8) & 0xFF) + (int)((h >> 16) & 0xFF) + (int)((h >> 24) & 0xFF) - 510;
}
__host__ __device__ __forceinline__ uint64_t list_of_row(uint64_t centroid_seed, uint64_t row, int nlist) {
  return mix64(centroid_seed ^ (row * 0xA0761D6478BD642Full) ^ 0x5851F42D4C957F2Dull) % (uint64_t)nlist;
}

template <typename OutT>
__device__ __forceinline__ OutT cast_out(float x);
template <>
__device__ __forceinline__ __half cast_out<__half>(float x) { return __float2half_rn(x); }
template <>
__device__ __forceinline__ float cast_out<float>(float x) { return x; }

// One warp per row.
template <typename OutT>
__global__ void synth_rows_kernel(OutT* __restrict__ out, int64_t n, int d, int64_t row0, b200_synth_spec spec) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t r = warp; r < n; r += nwarps) {
    const uint64_t row = (uint64_t)(row0 + r);
    const uint64_t rk = row_key(spec.seed, row);
    uint64_t ck = 0;
    if (spec.clustered) ck = row_key(spec.centroid_seed, list_of_row(spec.centroid_seed, row, spec.nlist));
    long long ss = 0;
    for (int j = lane; j < d; j += 32) {
      int v = noise_at(rk, j);
      if (spec.clustered) v = spec.cw * noise_at(ck, j) + spec.nw * v;
      ss += (long long)v * v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const double norm = sqrt((double)ss);
    OutT* orow = out + r * (int64_t)d;
    for (int j = lane; j < d; j += 32) {
      int v = noise_at(rk, j);
      if (spec.clustered) v = spec.cw * noise_at(ck, j) + spec.nw * v;
      float x = (ss == 0) ? 0.0f : (float)((double)v / norm);
      orow[j] = cast_out<OutT>(x);
    }
  }
}

// Same rows, written in a permuted order: out[p] = row (row0 + src_rows[p])  (IVF list order).
__global__ void synth_rows_indirect_kernel(__half* __restrict__ out, const uint32_t* __restrict__ src_rows, int64_t n,
                                           int d, int64_t row0, b200_synth_spec spec) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t p = warp; p < n; p += nwarps) {
    const uint64_t row = (uint64_t)(row0 + (int64_t)src_rows[p]);
    const uint64_t rk = row_key(spec.seed, row);
    uint64_t ck = 0;
    if (spec.clustered) ck = row_key(spec.centroid_seed, list_of_row(spec.centroid_seed, row, spec.nlist));
    long long ss = 0;
    for (int j = lane; j < d; j += 32) {
      int v = noise_at(rk, j);
      if (spec.clustered) v = spec.cw * noise_at(ck, j) + spec.nw * v;
      ss += (long long)v * v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const double norm = sqrt((double)ss);
    __half* orow = out + p * (int64_t)d;
    for (int j = lane; j < d; j += 32) {
      int v = noise_at(rk, j);
      if (spec.clustered) v = spec.cw * noise_at(ck, j) + spec.nw * v;
      orow[j] = __float2half_rn((ss == 0) ? 0.0f : (float)((double)v / norm));
    }
  }
}

int synth_rows_indirect_f16(__half* out, const uint32_t* src_rows, int64_t n, int d, int64_t row0,
                            const b200_synth_spec* spec, cudaStream_t st) {
  if (n == 0) return B200_OK;
  int64_t blocks = (n + 7) / 8;
  if (blocks > 132 * 32) blocks = 132 * 32;
  synth_rows_indirect_kernel<<<(unsigned)blocks, 256, 0, st>>>(out, src_rows, n, d, row0, *spec);
  B200_LAUNCH_OK();
  return B200_OK;
}

template <typename OutT>
int synth_rows(OutT* d_out, int64_t n, int d, int64_t row0, const b200_synth_spec* spec, cudaStream_t st) {
  B200_CHECK(spec != nullptr && d_out != nullptr, B200_ERR_INVALID, "synth_rows: null argument");
  B200_CHECK(n >= 0 && d > 0, B200_ERR_INVALID, "synth_rows: bad shape n=%lld d=%d", (long long)n, d);
  B200_CHECK(!spec->clustered || spec->nlist > 0, B200_ERR_INVALID, "synth_rows: clustered needs nlist > 0");
  if (n == 0) return B200_OK;
  const int threads = 256;
  int64_t blocks = (n + 7) / 8;
  if (blocks > 132 * 32) blocks = 132 * 32;
  synth_rows_kernel<OutT><<<(unsigned)blocks, threads, 0, st>>>(d_out, n, d, row0, *spec);
  B200_LAUNCH_OK();
  return B200_OK;
}

template int synth_rows<__half>(__half*, int64_t, int, int64_t, const b200_synth_spec*, cudaStream_t);
template int synth_rows<float>(float*, int64_t, int, int64_t, const b200_synth_spec*, cudaStream_t);

}  // namespace b200

extern "C" int b200_synth_rows_f16(void* d_out, int64_t n, int d, int64_t row0, const b200_synth_spec* spec, void* stream) {
  return b200::synth_rows<__half>((__half*)d_out, n, d, row0, spec, (cudaStream_t)stream);
}
extern "C" int b200_synth_rows_f32(float* d_out, int64_t n, int d, int64_t row0, const b200_synth_spec* spec, void* stream) {
  return b200::synth_rows<float>(d_out, n, d, row0, spec, (cudaStream_t)stream);
}
