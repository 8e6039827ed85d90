// Weight upload from b200_tensor_view lists (clip_model.cu, text_encoder.cu): look a tensor up by name, check its
// element count, convert to the device layout (bf16 round-to-nearest-even or fp32) and copy it to the device.
#pragma once
#include "common.cuh"
#include <cstring>
#include <map>
#include <string>
#include <vector>

namespace b200 {

static inline float view_get(const b200_tensor_view& v, size_t i) {
  if (v.dtype == 0) return ((const float*)v.data)[i];
  return __half2float(((const __half*)v.data)[i]);
}
static inline uint16_t f32_to_bf16_rn(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);  // NaN
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
static inline size_t view_count(const b200_tensor_view& v) {
  size_t n = 1;
  for (int i = 0; i < v.ndim; i++) n *= (size_t)v.shape[i];
  return n;
}

struct Loader {
  std::map<std::string, const b200_tensor_view*> by_name;
  std::vector<uint16_t> tmp16;
  std::vector<float> tmp32;
  // Indexes the caller's n views by name (they must outlive the loader); B200_ERR_INVALID for a malformed view.
  int index(const b200_tensor_view* views, int n) {
    for (int i = 0; i < n; i++) {
      B200_CHECK(views[i].name && views[i].data && (views[i].dtype == 0 || views[i].dtype == 1) && views[i].ndim >= 0 &&
                     views[i].ndim <= 4,
                 B200_ERR_INVALID, "load_weights: malformed tensor view %d", i);
      by_name[views[i].name] = &views[i];
    }
    return B200_OK;
  }
  const b200_tensor_view* find(const std::string& name, size_t count) {
    auto it = by_name.find(name);
    if (it == by_name.end()) { set_error("load_weights: tensor '%s' is missing", name.c_str()); return nullptr; }
    if (view_count(*it->second) != count) {
      set_error("load_weights: tensor '%s' has %zu elements, expected %zu", name.c_str(), view_count(*it->second), count);
      return nullptr;
    }
    return it->second;
  }
  // dst bf16 [rows, dst_ld] <- src [rows, cols] (zero padded columns keep their zeros)
  int put_bf16(const std::string& name, __nv_bfloat16* dst, size_t rows, size_t cols, size_t dst_ld) {
    const b200_tensor_view* v = find(name, rows * cols);
    if (!v) return B200_ERR_INVALID;
    tmp16.assign(rows * dst_ld, 0);
    for (size_t r = 0; r < rows; r++)
      for (size_t c = 0; c < cols; c++) tmp16[r * dst_ld + c] = f32_to_bf16_rn(view_get(*v, r * cols + c));
    B200_CUDA(cudaMemcpy(dst, tmp16.data(), tmp16.size() * 2, cudaMemcpyHostToDevice));
    return B200_OK;
  }
  // dst bf16 [rows, cols] <- the transpose of src [cols, rows] (a Linear weight into the [in, out] layout)
  int put_bf16_t(const std::string& name, __nv_bfloat16* dst, size_t src_rows, size_t src_cols) {
    const b200_tensor_view* v = find(name, src_rows * src_cols);
    if (!v) return B200_ERR_INVALID;
    tmp16.assign(src_rows * src_cols, 0);
    for (size_t r = 0; r < src_rows; r++)
      for (size_t c = 0; c < src_cols; c++) tmp16[c * src_rows + r] = f32_to_bf16_rn(view_get(*v, r * src_cols + c));
    B200_CUDA(cudaMemcpy(dst, tmp16.data(), tmp16.size() * 2, cudaMemcpyHostToDevice));
    return B200_OK;
  }
  int put_f32(const std::string& name, float* dst, size_t count) {
    const b200_tensor_view* v = find(name, count);
    if (!v) return B200_ERR_INVALID;
    tmp32.resize(count);
    for (size_t i = 0; i < count; i++) tmp32[i] = view_get(*v, i);
    B200_CUDA(cudaMemcpy(dst, tmp32.data(), count * 4, cudaMemcpyHostToDevice));
    return B200_OK;
  }
};

}  // namespace b200
