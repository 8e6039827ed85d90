// Copying a built index back to the host, for writing it out as a FAISS file (faiss_io.write_index): the quantiser
// parameters, and the row / code store a slot range at a time, so a writer's host memory stays bounded by its chunk.
#include "index.cuh"
#include <vector>

using namespace b200;

extern "C" {

int b200_index_get_quantizer(b200_index* idx, float* h_centroids, float* h_codebook, float* h_A, float* h_b,
                             int32_t* h_info) {
  B200_CHECK(idx, B200_ERR_INVALID, "get_quantizer: null index");
  DeviceGuard g(idx->device);
  std::lock_guard<std::mutex> lock(idx->mu);
  const int d = idx->d;
  if (h_info) {
    const int32_t info[8] = {idx->nlist, idx->pq_M, idx->pq_by_residual ? 1 : 0, idx->pt_A ? 1 : 0, idx->pt_b ? 1 : 0,
                             d, idx->d_in, idx->nprobe};
    for (int i = 0; i < 8; i++) h_info[i] = info[i];
  }
  if (h_centroids && idx->nlist > 0) {
    const size_t count = (size_t)idx->nlist * d;
    if (idx->pq_M > 0) {
      B200_CUDA(cudaMemcpy(h_centroids, idx->pq_centroids, count * 4, cudaMemcpyDeviceToHost));
    } else {
      std::vector<__half> tmp(count);
      B200_CUDA(cudaMemcpy(tmp.data(), idx->centroids, count * 2, cudaMemcpyDeviceToHost));
      for (size_t i = 0; i < count; i++) h_centroids[i] = __half2float(tmp[i]);
    }
  }
  if (h_codebook && idx->pq_M > 0)
    B200_CUDA(cudaMemcpy(h_codebook, idx->pq_codebook, (size_t)256 * d * 4, cudaMemcpyDeviceToHost));
  if (h_A && idx->pt_A) B200_CUDA(cudaMemcpy(h_A, idx->pt_A, (size_t)d * idx->d_in * 4, cudaMemcpyDeviceToHost));
  if (h_b && idx->pt_b) B200_CUDA(cudaMemcpy(h_b, idx->pt_b, (size_t)d * 4, cudaMemcpyDeviceToHost));
  return B200_OK;
}

int b200_index_copy_rows(b200_index* idx, int64_t s0, int64_t n, void* h_rows, int64_t* h_ids) {
  B200_CHECK(idx && s0 >= 0 && n >= 0, B200_ERR_INVALID, "copy_rows: bad argument");
  DeviceGuard g(idx->device);
  B200_CHECK(!idx->host, B200_ERR_UNSUPPORTED, "copy_rows: the lists are in host memory (the file they came from)");
  if (idx->nlist > 0) B200_TRY(ivf_finalize(idx));
  B200_CHECK(s0 + n <= idx->ntotal, B200_ERR_INVALID, "copy_rows: slots [%lld, %lld) past the %lld stored rows",
             (long long)s0, (long long)(s0 + n), (long long)idx->ntotal);
  if (n == 0) return B200_OK;
  std::lock_guard<std::mutex> lock(idx->mu);
  const size_t width = idx->pq_M > 0 ? (size_t)idx->pq_M : (size_t)idx->d * 2;
  const size_t pitch = (size_t)idx->row_bytes;
  if (h_rows)
    B200_CUDA(cudaMemcpy2D(h_rows, width, reinterpret_cast<const uint8_t*>(idx->rows) + (size_t)s0 * pitch, pitch, width,
                           (size_t)n, cudaMemcpyDeviceToHost));
  if (h_ids) {
    if (idx->nlist > 0) {
      std::vector<uint32_t> tmp((size_t)n);
      B200_CUDA(cudaMemcpy(tmp.data(), idx->row_ids + s0, (size_t)n * 4, cudaMemcpyDeviceToHost));
      for (int64_t i = 0; i < n; i++) h_ids[i] = idx->id_base + (int64_t)tmp[i];
    } else {
      for (int64_t i = 0; i < n; i++) h_ids[i] = idx->id_base + s0 + i;
    }
  }
  return B200_OK;
}

}  // extern "C"
