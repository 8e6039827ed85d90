// Row-scan building blocks shared by the flat (knn_scan.cu), IVF-Flat (knn_ivf.cu) and IVF-PQ (knn_ivfpq.cu)
// kernels: the query slice a lane keeps in registers, the fp16-chunk dot product, the offer of a warp's scores to
// its candidate lists, the range-hit append and the row range of a list segment.
#pragma once
#include "topk.cuh"

namespace b200 {

// This lane's slice of one fp32 query: chunks lane, lane+32, ... (8 columns per chunk), zero past `cpr`.
template <int CH>
__device__ __forceinline__ void load_query_slice(float (&qr)[CH][8], const float* q, int cpr, int lane, bool valid) {
#pragma unroll
  for (int c = 0; c < CH; c++) {
    const int ci = c * 32 + lane;
    if (valid && ci < cpr) {
      const float4 a = *reinterpret_cast<const float4*>(q + ci * 8);
      const float4 b = *reinterpret_cast<const float4*>(q + ci * 8 + 4);
      qr[c][0] = a.x; qr[c][1] = a.y; qr[c][2] = a.z; qr[c][3] = a.w;
      qr[c][4] = b.x; qr[c][5] = b.y; qr[c][6] = b.z; qr[c][7] = b.w;
    } else {
#pragma unroll
      for (int j = 0; j < 8; j++) qr[c][j] = 0.0f;
    }
  }
}

// One 16-byte chunk of an fp16 row as eight fp32 values.
__device__ __forceinline__ void chunk_to_f32(uint4 v, float (&f)[8]) {
  const __half2* h2 = reinterpret_cast<const __half2*>(&v);
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const float2 t = __half22float2(h2[j]);
    f[2 * j] = t.x; f[2 * j + 1] = t.y;
  }
}
// acc += <chunk, qr>: one fmaf per element, elements in ascending order.  Every scan sums a row this way, chunk
// after chunk, which is what makes their scores equal bit for bit.
__device__ __forceinline__ void fma_chunk(const float (&f)[8], const float (&qr)[8], float& acc) {
#pragma unroll
  for (int j = 0; j < 8; j++) acc = fmaf(f[j], qr[j], acc);
}
__device__ __forceinline__ void fma_chunk(uint4 v, const float (&qr)[8], float& acc) {
  const __half2* h2 = reinterpret_cast<const __half2*>(&v);
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const float2 t = __half22float2(h2[j]);
    acc = fmaf(t.x, qr[2 * j], acc);
    acc = fmaf(t.y, qr[2 * j + 1], acc);
  }
}

// Offer the warp's keys to its replace-worst lists: lanes with `offer` set are taken in lane order and their key
// is inserted by the whole warp.  `wkeys` holds NQ lists of k keys; the popping lane's value index (lane >> SH)
// selects the list, as laid out by warp_transpose_reduce.  One list: NQ = 1.
template <int NQ = 1, int SH = 0>
__device__ __forceinline__ void warp_offer(unsigned long long* wkeys, int k, bool offer, unsigned long long key,
                                           unsigned long long* worst, int* worst_pos, int lane) {
  unsigned pend = __ballot_sync(FULL, offer);
  while (pend) {
    const int src = __ffs(pend) - 1;
    pend &= pend - 1;
    const unsigned long long ckey = __shfl_sync(FULL, key, src);
    const int cq = (src >> SH) % NQ;
#pragma unroll
    for (int q = 0; q < NQ; q++)
      if (cq == q) warp_list_insert(wkeys + q * k, k, ckey, worst[q], worst_pos[q], lane);
  }
}

// Empty the warp's lists before a scan / copy one of them out after it (the caller orders them with __syncwarp).
__device__ __forceinline__ void warp_lists_clear(unsigned long long* wkeys, int count, int lane) {
  for (int i = lane; i < count; i += 32) wkeys[i] = 0ull;
}
__device__ __forceinline__ void warp_list_store(unsigned long long* out, const unsigned long long* list, int k, int lane) {
  for (int j = lane; j < k; j += 32) out[j] = list[j];
}

// Range search: append a hit to the query's global list; the counter keeps counting past `cap`.
__device__ __forceinline__ void range_append(unsigned long long* out, unsigned int cap, unsigned int* counter, float score,
                                             uint32_t row) {
  const unsigned int pos = atomicAdd(counter, 1u);
  if (pos < cap) out[pos] = make_key(score, row);
}

// Rows [beg, end) of segment `seg` of `segs` equal segments of list `list`, segment length rounded up to `align`.
__device__ __forceinline__ void segment_rows(const int64_t* offsets, uint32_t list, int segs, int seg, int align, int64_t& beg,
                                             int64_t& end) {
  const int64_t lbeg = offsets[list], lend = offsets[list + 1];
  const int64_t per = ((lend - lbeg + segs - 1) / segs + align - 1) / align * align;
  beg = lbeg + (int64_t)seg * per;
  end = beg + per < lend ? beg + per : lend;
}

}  // namespace b200
