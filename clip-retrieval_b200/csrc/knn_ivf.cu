// Search path, IVF-Flat (SURVEY.md §2.2 S2): inner-product IVF over fp16 rows with the knob the
// reference touches through faiss.extract_index_ivf(index).nprobe (clip_back.py:357-361,368-369).
//
// Layout in HBM: rows are stored LIST AFTER LIST (`rows`, fp16 [ntotal, d]) with `list_offsets`
// [nlist+1] and `row_ids` (slot -> insertion id), so a probed list is one contiguous stream; its inverse
// `id_to_slot` is rebuilt whenever the store changes (finalize, add_synthetic), never during a search.
// Search = (1) coarse: the flat scan kernel over the centroid matrix with k = nprobe;
//          (2) list scan: one CTA per (query, probe, segment) streams its slice of the list with the
//              same warp-per-row 128-bit loads / fp32 FMA / per-warp replace-worst lists as the flat
//              scan; (3) the chunked bitonic select over the per-warp candidates of each query.
// List-scan keys carry the insertion id (row_ids[slot]), not the slot, so equal scores come back in
// ascending id order even when the tied rows sit in different lists (explicit lists of an index file).
// HBM-bound: bytes per query = nprobe * (N/nlist) * d * 2 (+ nlist * d * 2 for the coarse step).
#include "index.cuh"
#include "scan.cuh"
#include <cub/cub.cuh>
#include <algorithm>

namespace b200 {

constexpr int SCAN_ALIGN = 4;

// ---- assignment: argmax_c <x, c> --------------------------------------------------------------------
// One warp per row; the row sits in registers (fp32), centroids stream from L2.
template <int CH>
__global__ void __launch_bounds__(256)
ivf_assign_kernel(const uint4* __restrict__ X, int64_t n, int cpr, const uint4* __restrict__ Cn, int nlist,
                  uint32_t* __restrict__ assign) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  float x[CH][8];
#pragma unroll
  for (int c = 0; c < CH; c++) {
    const int ci = c * 32 + lane;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (ci < cpr) v = X[row * cpr + ci];
    chunk_to_f32(v, x[c]);
  }
  float best = -INFINITY;
  uint32_t best_l = 0;
  for (int l0 = 0; l0 < nlist; l0 += 4) {
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int u = 0; u < 4; u++) {
      if (l0 + u < nlist) {
#pragma unroll
        for (int c = 0; c < CH; c++) {
          const int ci = c * 32 + lane;
          if (ci < cpr) fma_chunk(Cn[(int64_t)(l0 + u) * cpr + ci], x[c], acc[u]);
        }
      }
    }
    warp_transpose_reduce<4>(acc, lane);  // lane L holds list l0 + (L >> 3)
    const int li = l0 + (lane >> 3);
    float s = li < nlist ? acc[0] : -INFINITY;
    uint32_t sl = (uint32_t)li;
    // max over the four candidates, ties to the lower list id
#pragma unroll
    for (int o = 16; o >= 8; o >>= 1) {
      const float os = __shfl_xor_sync(FULL, s, o);
      const uint32_t ol = __shfl_xor_sync(FULL, sl, o);
      if (os > s || (os == s && ol < sl)) { s = os; sl = ol; }
    }
    if (s > best) { best = s; best_l = sl; }
  }
  if (lane == 0) assign[row] = best_l;
}

__global__ void lists_by_construction_kernel(uint32_t* __restrict__ lists, uint32_t* __restrict__ idx, int64_t n,
                                             int64_t row0, uint64_t centroid_seed, int nlist) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t z = centroid_seed ^ ((uint64_t)(row0 + i) * 0xA0761D6478BD642Full) ^ 0x5851F42D4C957F2Dull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z = z ^ (z >> 31);
  lists[i] = (uint32_t)(z % (uint64_t)nlist);
  idx[i] = (uint32_t)i;
}

__global__ void apply_explicit_lists_kernel(const uint32_t* __restrict__ explicit_lists, int64_t n, uint32_t* __restrict__ lists) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && explicit_lists[i] != 0xFFFFFFFFu) lists[i] = explicit_lists[i];
}

__global__ void invert_ids_kernel(const uint32_t* __restrict__ row_ids, int64_t n, uint32_t* __restrict__ id_to_slot) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) id_to_slot[row_ids[i]] = (uint32_t)i;
}

__global__ void iota_kernel(uint32_t* __restrict__ idx, int64_t n, uint32_t base) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) idx[i] = base + (uint32_t)i;
}

// list id of every already-bucketed slot (expands list_offsets)
__global__ void expand_offsets_kernel(const int64_t* __restrict__ offsets, int nlist, uint32_t* __restrict__ lists) {
  const int l = blockIdx.x;
  for (int64_t i = offsets[l] + threadIdx.x; i < offsets[l + 1]; i += blockDim.x) lists[i] = (uint32_t)l;
}

__global__ void offsets_from_sorted_kernel(const uint32_t* __restrict__ sorted_lists, int64_t n, int nlist,
                                           int64_t* __restrict__ offsets) {
  // offsets[l] = first position whose list >= l  (binary search per list)
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l > nlist) return;
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (sorted_lists[mid] < (uint32_t)l) lo = mid + 1; else hi = mid;
  }
  offsets[l] = lo;
}

// gather rows into list order: src slot < nold comes from `old_rows`, else from `new_rows`
__global__ void gather_sorted_rows_kernel(const uint4* __restrict__ old_rows, const uint4* __restrict__ new_rows,
                                          int64_t nold, const uint32_t* __restrict__ src, int64_t n, int cpr,
                                          uint4* __restrict__ dst, const uint32_t* __restrict__ old_ids,
                                          uint32_t* __restrict__ new_ids) {
  const int lane = threadIdx.x & 31;
  const int64_t p = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (p >= n) return;
  const uint32_t s = src[p];
  const uint4* from = s < nold ? old_rows + (int64_t)s * cpr : new_rows + (int64_t)(s - nold) * cpr;
  for (int c = lane; c < cpr; c += 32) dst[p * cpr + c] = from[c];
  if (lane == 0) new_ids[p] = s < nold ? old_ids[s] : s;  // pending rows: slot index == insertion id
}

// generate synthetic rows straight into list order
__global__ void sorted_src_to_ids_kernel(const uint32_t* __restrict__ src, int64_t n, uint32_t base, uint32_t* ids) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) ids[i] = base + src[i];
}

// ---- list scan ---------------------------------------------------------------------------------------
template <int CH>
__global__ void __launch_bounds__(256)
ivf_scan_kernel(const uint4* __restrict__ X, const uint32_t* __restrict__ row_ids, int cpr, const float* __restrict__ Q,
                const unsigned long long* __restrict__ probes, int nprobe, int segs, const int64_t* __restrict__ offsets,
                int k, unsigned long long* __restrict__ out_keys, int64_t out_stride_q) {
  extern __shared__ unsigned long long s_keys[];  // [warps][k]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int seg = blockIdx.x % segs;
  const int p = (blockIdx.x / segs) % nprobe;
  const int q = blockIdx.x / (segs * nprobe);
  unsigned long long* wkeys = s_keys + (size_t)warp * k;
  warp_lists_clear(wkeys, k, lane);
  __syncwarp();
  const unsigned long long pk = probes[(int64_t)q * nprobe + p];
  unsigned long long worst = 0ull;
  int worst_pos = 0;
  if (pk != 0ull) {
    int64_t beg, end;
    segment_rows(offsets, key_id(pk), segs, seg, SCAN_ALIGN, beg, end);
    const int d = cpr * 8;
    float qr[CH][8];
    load_query_slice<CH>(qr, Q + (size_t)q * d, cpr, lane, true);
    for (int64_t r0 = beg + (int64_t)warp * 4; r0 < end; r0 += (int64_t)nwarps * 4) {
      uint4 v[4][CH];
#pragma unroll
      for (int u = 0; u < 4; u++) {
#pragma unroll
        for (int c = 0; c < CH; c++) {
          const int ci = c * 32 + lane;
          if (r0 + u < end && ci < cpr) v[u][c] = ld_nc_v4(X + (r0 + u) * cpr + ci);
          else v[u][c] = make_uint4(0u, 0u, 0u, 0u);
        }
      }
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int u = 0; u < 4; u++) {
#pragma unroll
        for (int c = 0; c < CH; c++) fma_chunk(v[u][c], qr[c], acc[u]);
      }
      warp_transpose_reduce<4>(acc, lane);
      const float s = acc[0];
      const int64_t my_r = r0 + (lane >> 3);
      const bool live = ((lane & 7) == 0) && my_r < end && (s == s);
      // Only a row scoring at least the worst kept score can enter the list; the insertion id that breaks its
      // ties is loaded for those rows alone (every row while the list fills, rarely after).
      const bool reach = live && f32_to_ordered(s) >= (uint32_t)(worst >> 32);
      unsigned long long key = 0ull;
      if (reach) key = make_key(s, __ldg(row_ids + my_r));
      warp_offer(wkeys, k, reach && key > worst, key, &worst, &worst_pos, lane);
    }
  }
  __syncwarp();
  warp_list_store(out_keys + (int64_t)q * out_stride_q + ((int64_t)(p * segs + seg) * nwarps + warp) * k, wkeys, k, lane);
}

typedef void (*ivf_scan_fn)(const uint4*, const uint32_t*, int, const float*, const unsigned long long*, int, int,
                            const int64_t*, int, unsigned long long*, int64_t);
static ivf_scan_fn pick_ivf_scan(int ch) {
  switch (ch) {
    case 1: return ivf_scan_kernel<1>;
    case 2: return ivf_scan_kernel<2>;
    case 3: return ivf_scan_kernel<3>;
    case 4: return ivf_scan_kernel<4>;
    case 5: return ivf_scan_kernel<5>;
    case 6: return ivf_scan_kernel<6>;
    case 7: return ivf_scan_kernel<7>;
    case 8: return ivf_scan_kernel<8>;
  }
  return nullptr;
}
typedef void (*ivf_assign_fn)(const uint4*, int64_t, int, const uint4*, int, uint32_t*);
static ivf_assign_fn pick_ivf_assign(int ch) {
  switch (ch) {
    case 1: return ivf_assign_kernel<1>;
    case 2: return ivf_assign_kernel<2>;
    case 3: return ivf_assign_kernel<3>;
    case 4: return ivf_assign_kernel<4>;
    case 5: return ivf_assign_kernel<5>;
    case 6: return ivf_assign_kernel<6>;
    case 7: return ivf_assign_kernel<7>;
    case 8: return ivf_assign_kernel<8>;
  }
  return nullptr;
}

// ---- host side ----------------------------------------------------------------------------------------

int ivf_create(b200_index* idx, int nlist, const float* h_centroids) {
  idx->nlist = nlist;
  idx->nprobe = 1;
  if (h_centroids) {   // IVF-PQ passes none: its coarse step and dis0 use the fp32 centroids (knn_ivfpq.cu)
    const size_t count = (size_t)nlist * idx->d;
    B200_CUDA(cudaMalloc((void**)&idx->centroids, count * sizeof(__half)));
    std::vector<__half> tmp(count);
    for (size_t i = 0; i < count; i++) tmp[i] = __float2half_rn(h_centroids[i]);
    B200_CUDA(cudaMemcpy(idx->centroids, tmp.data(), count * sizeof(__half), cudaMemcpyHostToDevice));
  }
  B200_CUDA(cudaMalloc((void**)&idx->list_offsets, (size_t)(nlist + 1) * sizeof(int64_t)));
  B200_CUDA(cudaMemset(idx->list_offsets, 0, (size_t)(nlist + 1) * sizeof(int64_t)));
  idx->h_list_offsets.assign(nlist + 1, 0);
  return B200_OK;
}

void ivf_free(b200_index* idx) {
  if (idx->centroids) cudaFree(idx->centroids);
  if (idx->list_offsets) cudaFree(idx->list_offsets);
  if (idx->row_ids) cudaFree(idx->row_ids);
  if (idx->pending) cudaFree(idx->pending);
  if (idx->id_to_slot) cudaFree(idx->id_to_slot);
  if (idx->pq_centroids) cudaFree(idx->pq_centroids);
  if (idx->pq_codebook) cudaFree(idx->pq_codebook);
  if (idx->pt_A) cudaFree(idx->pt_A);
  if (idx->pt_b) cudaFree(idx->pt_b);
  host_lists_free(idx);
}

int grow_pending(b200_index* idx, int64_t need, bool amortised) {
  if (need <= idx->pending_cap) return B200_OK;
  const int64_t rb = idx->row_bytes;
  const int64_t cap = amortised ? std::max(need, idx->pending_cap + idx->pending_cap / 2) : need;
  void* np = nullptr;
  B200_CUDA(cudaMalloc(&np, (size_t)cap * rb));
  if (idx->pending) {
    B200_CUDA(cudaMemcpy(np, idx->pending, (size_t)idx->npending * rb, cudaMemcpyDeviceToDevice));
    B200_CUDA(cudaFree(idx->pending));
  }
  idx->pending = (__half*)np;
  idx->pending_cap = cap;
  return B200_OK;
}

// Sort (list, src) pairs by list (stable) into (lists2, src2) and derive offsets [nlist + 1] from the sorted lists.
// As with cub, a null `tmp` only reports the scratch size in tmp_bytes.
static int sort_pairs_by_list(void* tmp, size_t& tmp_bytes, uint32_t* lists, uint32_t* lists2, uint32_t* src,
                              uint32_t* src2, int64_t n, int nlist, int64_t* offsets) {
  int bits = 1;
  while ((1ll << bits) < nlist) bits++;
  cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, lists, lists2, src, src2, (int)n, 0, bits);
  if (!tmp) return B200_OK;
  count_launch(4);
  offsets_from_sorted_kernel<<<(nlist + 1 + 255) / 256, 256>>>(lists2, n, nlist, offsets);
  B200_LAUNCH_OK();
  return B200_OK;
}

// The index's own lists: sorts into fresh arrays, sets idx->list_offsets; the caller frees *sorted_src.
static int sort_by_list(b200_index* idx, uint32_t* lists, uint32_t* src, int64_t n, uint32_t** sorted_src) {
  uint32_t *lists2 = nullptr, *src2 = nullptr;
  B200_CUDA(cudaMalloc((void**)&lists2, (size_t)n * 4));
  B200_CUDA(cudaMalloc((void**)&src2, (size_t)n * 4));
  B200_CHECK(n < (1ll << 31), B200_ERR_UNSUPPORTED, "ivf: at most 2^31 rows per finalize");
  size_t tmp_bytes = 0;
  void* tmp = nullptr;
  B200_TRY(sort_pairs_by_list(nullptr, tmp_bytes, lists, lists2, src, src2, n, idx->nlist, idx->list_offsets));
  B200_CUDA(cudaMalloc(&tmp, tmp_bytes));
  B200_TRY(sort_pairs_by_list(tmp, tmp_bytes, lists, lists2, src, src2, n, idx->nlist, idx->list_offsets));
  B200_CUDA(cudaDeviceSynchronize());
  B200_CUDA(cudaFree(tmp));
  B200_CUDA(cudaFree(lists2));
  *sorted_src = src2;
  return B200_OK;
}

static int refresh_host_offsets(b200_index* idx) {
  B200_CUDA(cudaMemcpy(idx->h_list_offsets.data(), idx->list_offsets, (size_t)(idx->nlist + 1) * 8, cudaMemcpyDeviceToHost));
  idx->max_list = 0;
  for (int l = 0; l < idx->nlist; l++)
    idx->max_list = std::max<int64_t>(idx->max_list, idx->h_list_offsets[l + 1] - idx->h_list_offsets[l]);
  return B200_OK;
}

// id -> slot: the inverse of row_ids, for reconstruct-by-id and for the rows of search_and_reconstruct.  Built
// whenever the store changes so that a search (possibly under CUDA-graph capture) never allocates it.
static int build_id_to_slot(b200_index* idx) {
  if (idx->id_to_slot) B200_CUDA(cudaFree(idx->id_to_slot));
  idx->id_to_slot = nullptr;
  if (idx->ntotal == 0) return B200_OK;
  B200_CUDA(cudaMalloc((void**)&idx->id_to_slot, (size_t)idx->ntotal * 4));
  invert_ids_kernel<<<(unsigned)((idx->ntotal + 255) / 256), 256>>>(idx->row_ids, idx->ntotal, idx->id_to_slot);
  B200_LAUNCH_OK();
  B200_CUDA(cudaDeviceSynchronize());
  return B200_OK;
}

// Rows are moved as row_bytes / 16 chunks of 16 bytes: fp16 rows (IVF-Flat) and padded code rows (IVF-PQ) alike.
// IVF-PQ rows always carry an explicit list, so only IVF-Flat rows are assigned by inner product.
int ivf_finalize(b200_index* idx) {
  if (idx->npending == 0) return B200_OK;
  const int d = idx->d, ch = (d / 8 + 31) / 32;
  const int64_t rb = idx->row_bytes, cpr = rb / 16;
  const int64_t nold = idx->ntotal, nnew = idx->npending, n = nold + nnew;
  B200_CHECK(n < (1ll << 32), B200_ERR_UNSUPPORTED, "ivf: a shard holds at most 2^32 rows");
  uint32_t *lists = nullptr, *src = nullptr;
  B200_CUDA(cudaMalloc((void**)&lists, (size_t)n * 4));
  B200_CUDA(cudaMalloc((void**)&src, (size_t)n * 4));
  if (nold > 0) {
    expand_offsets_kernel<<<idx->nlist, 256>>>(idx->list_offsets, idx->nlist, lists);
    B200_LAUNCH_OK();
  }
  if (idx->pq_M == 0) {
    ivf_assign_fn afn = pick_ivf_assign(ch);
    B200_CHECK(afn != nullptr, B200_ERR_UNSUPPORTED, "ivf: unsupported dimension %d", d);
    afn<<<(unsigned)((nnew + 7) / 8), 256>>>(reinterpret_cast<const uint4*>(idx->pending), nnew, d / 8,
                                             reinterpret_cast<const uint4*>(idx->centroids), idx->nlist, lists + nold);
    B200_LAUNCH_OK();
  }
  if (!idx->pending_lists.empty()) {
    // rows added with an explicit list (an index file's own inverted lists) keep it
    idx->pending_lists.resize((size_t)nnew, 0xFFFFFFFFu);
    uint32_t* d_explicit = nullptr;
    B200_CUDA(cudaMalloc((void**)&d_explicit, (size_t)nnew * 4));
    B200_CUDA(cudaMemcpy(d_explicit, idx->pending_lists.data(), (size_t)nnew * 4, cudaMemcpyHostToDevice));
    apply_explicit_lists_kernel<<<(unsigned)((nnew + 255) / 256), 256>>>(d_explicit, nnew, lists + nold);
    B200_LAUNCH_OK();
    B200_CUDA(cudaDeviceSynchronize());
    B200_CUDA(cudaFree(d_explicit));
    idx->pending_lists.clear();
  }
  iota_kernel<<<(unsigned)((n + 255) / 256), 256>>>(src, n, 0u);
  B200_LAUNCH_OK();
  uint32_t* sorted_src = nullptr;
  B200_TRY(sort_by_list(idx, lists, src, n, &sorted_src));
  __half* nrows = nullptr;
  uint32_t* nids = nullptr;
  B200_CUDA(cudaMalloc((void**)&nrows, (size_t)n * rb));
  B200_CUDA(cudaMalloc((void**)&nids, (size_t)n * 4));
  gather_sorted_rows_kernel<<<(unsigned)((n + 7) / 8), 256>>>(
      reinterpret_cast<const uint4*>(idx->rows), reinterpret_cast<const uint4*>(idx->pending), nold, sorted_src, n, (int)cpr,
      reinterpret_cast<uint4*>(nrows), idx->row_ids, nids);
  B200_LAUNCH_OK();
  B200_CUDA(cudaDeviceSynchronize());
  B200_CUDA(cudaFree(sorted_src));
  B200_CUDA(cudaFree(lists));
  B200_CUDA(cudaFree(src));
  if (idx->rows) B200_CUDA(cudaFree(idx->rows));
  if (idx->row_ids) B200_CUDA(cudaFree(idx->row_ids));
  B200_CUDA(cudaFree(idx->pending));
  idx->pending = nullptr;
  idx->pending_cap = 0;
  idx->npending = 0;
  idx->rows = nrows;
  idx->row_ids = nids;
  idx->capacity = n;
  idx->ntotal = n;
  B200_TRY(build_id_to_slot(idx));
  return refresh_host_offsets(idx);
}

// Benchmark shortcut (SURVEY.md §8d row 4): rows of a clustered synthetic set whose nlist equals the
// index's are bucketed by their generating list and generated straight into list order.
int ivf_add_synthetic(b200_index* idx, int64_t n, int64_t row0, const b200_synth_spec* spec) {
  const int d = idx->d;
  const bool by_construction = spec->clustered && spec->nlist == idx->nlist && idx->ntotal == 0 && idx->npending == 0;
  if (!by_construction) {
    // general path: generate in insertion order, bucket at finalize by argmax inner product
    B200_TRY(grow_pending(idx, idx->npending + n, false));
    B200_TRY(synth_rows<__half>(idx->pending + idx->npending * d, n, d, row0, spec, 0));
    B200_CUDA(cudaDeviceSynchronize());
    idx->npending += n;
    return B200_OK;
  }
  B200_CHECK(n < (1ll << 31), B200_ERR_UNSUPPORTED, "ivf: at most 2^31 rows per add");
  uint32_t *lists = nullptr, *src = nullptr;
  B200_CUDA(cudaMalloc((void**)&lists, (size_t)n * 4));
  B200_CUDA(cudaMalloc((void**)&src, (size_t)n * 4));
  lists_by_construction_kernel<<<(unsigned)((n + 255) / 256), 256>>>(lists, src, n, row0, spec->centroid_seed, spec->nlist);
  B200_LAUNCH_OK();
  uint32_t* sorted_src = nullptr;
  B200_TRY(sort_by_list(idx, lists, src, n, &sorted_src));
  B200_CUDA(cudaFree(lists));
  B200_CUDA(cudaFree(src));
  B200_CUDA(cudaMalloc((void**)&idx->rows, (size_t)n * d * 2));
  B200_CUDA(cudaMalloc((void**)&idx->row_ids, (size_t)n * 4));
  // one synth launch per run of consecutive source rows would be wasteful: generate row by row id
  // rows[p] = synthetic row (row0 + sorted_src[p])
  B200_TRY(synth_rows_indirect_f16(idx->rows, sorted_src, n, d, row0, spec, 0));
  sorted_src_to_ids_kernel<<<(unsigned)((n + 255) / 256), 256>>>(sorted_src, n, 0u, idx->row_ids);
  B200_LAUNCH_OK();
  B200_CUDA(cudaDeviceSynchronize());
  B200_CUDA(cudaFree(sorted_src));
  idx->ntotal = n;
  idx->capacity = n;
  B200_TRY(build_id_to_slot(idx));
  return refresh_host_offsets(idx);
}

int ivf_lists(b200_index* idx, int64_t* h_sizes, int64_t* h_ids) {
  if (idx->host) return ivfpq_stream_lists(idx, h_sizes, h_ids);
  for (int l = 0; l < idx->nlist; l++) h_sizes[l] = idx->h_list_offsets[l + 1] - idx->h_list_offsets[l];
  if (h_ids && idx->ntotal > 0) {
    std::vector<uint32_t> tmp((size_t)idx->ntotal);
    B200_CUDA(cudaMemcpy(tmp.data(), idx->row_ids, (size_t)idx->ntotal * 4, cudaMemcpyDeviceToHost));
    for (int64_t i = 0; i < idx->ntotal; i++) h_ids[i] = idx->id_base + (int64_t)tmp[i];
  }
  return B200_OK;
}

int ivf_search_keys(b200_index* idx, const float* d_q, int nq, int k, unsigned long long* d_keys, cudaStream_t st) {
  const int d = idx->d, cpr = d / 8, ch = (cpr + 31) / 32;
  const int nprobe = std::min(idx->nprobe, idx->nlist);
  // (1) coarse quantiser: exhaustive scan of the centroids, k = nprobe
  void* ws = nullptr;
  B200_TRY(index_ws(idx, 3, (size_t)nq * nprobe * 8, &ws));
  unsigned long long* probes = (unsigned long long*)ws;
  const int coarse_launches0 = idx->last_scan_launches;
  B200_TRY(scan_topk_keys(idx, idx->centroids, idx->nlist, d_q, nq, nprobe, probes, st));
  idx->last_scan_launches = coarse_launches0;  // report list-scan launches only
  idx->ev_used = 0;
  // (2) list scan
  int threads = 256;
  while (threads > 64 && (size_t)(threads / 32) * k * 8 > 160 * 1024) threads >>= 1;
  const size_t smem = (size_t)(threads / 32) * k * 8;
  B200_CHECK(smem <= 200 * 1024, B200_ERR_UNSUPPORTED, "search: k=%d exceeds the supported maximum (8192)", k);
  ivf_scan_fn fn = pick_ivf_scan(ch);
  B200_CHECK(fn != nullptr, B200_ERR_UNSUPPORTED, "ivf: unsupported dimension %d", d);
  if (smem > 48 * 1024) B200_CUDA(cudaFuncSetAttribute((const void*)fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int nwarps = threads / 32;
  const int QB = 256;  // queries per batch (bounds the scratch)
  for (int q0 = 0; q0 < nq; q0 += QB) {
    const int qb = std::min(QB, nq - q0);
    // enough CTAs to fill the chip twice, segments no shorter than ~256 rows
    const int segs = list_segments(idx, 2 * idx->sms, (int64_t)qb * nprobe, 256);
    const int64_t M = (int64_t)nprobe * segs * nwarps * k;
    SelectPlan sel;
    B200_TRY(plan_select(M, k, &sel));
    void* w0 = nullptr;
    B200_TRY(index_ws(idx, 0, sel.keys(qb) * 8, &w0));
    unsigned long long* k1 = (unsigned long long*)w0;
    unsigned long long* k2 = k1 + (size_t)qb * M;
    B200_TRY(scan_timer_begin(idx, st));
    fn<<<(unsigned)((int64_t)qb * nprobe * segs), threads, smem, st>>>(
        reinterpret_cast<const uint4*>(idx->rows), idx->row_ids, cpr, d_q + (size_t)q0 * d, probes + (size_t)q0 * nprobe,
        nprobe, segs, idx->list_offsets, k, k1, M);
    B200_LAUNCH_OK();
    B200_TRY(scan_timer_end(idx, st));
    idx->last_scan_launches++;
    B200_TRY(select_topk(sel, k1, k2, d_keys + (size_t)q0 * k, qb, st));
  }
  return B200_OK;
}

// ---- range search over the probed lists (index.range_search on an IVF index: clip_filter.py:52) -----------
// FAISS IndexIVF::range_search visits the nprobe lists of the query and reports every row whose inner product
// exceeds the threshold.  One CTA per (probe, segment); hits are appended as (score, slot) keys (decoded to ids
// through row_ids; the host sorts the hits by id, so no tie order is needed here).
template <int CH>
__global__ void __launch_bounds__(256)
ivf_range_kernel(const uint4* __restrict__ X, int cpr, const float* __restrict__ Q, const unsigned long long* __restrict__ probes,
                 int nprobe, int segs, const int64_t* __restrict__ offsets, float thresh, unsigned long long* __restrict__ out,
                 unsigned int cap, unsigned int* __restrict__ counter) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int seg = blockIdx.x % segs;
  const int p = blockIdx.x / segs;
  const unsigned long long pk = probes[p];
  if (pk == 0ull) return;
  int64_t beg, end;
  segment_rows(offsets, key_id(pk), segs, seg, SCAN_ALIGN, beg, end);
  float qr[CH][8];
  load_query_slice<CH>(qr, Q, cpr, lane, true);
  for (int64_t r0 = beg + (int64_t)warp * 4; r0 < end; r0 += (int64_t)nwarps * 4) {
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int u = 0; u < 4; u++) {
#pragma unroll
      for (int c = 0; c < CH; c++) {
        const int ci = c * 32 + lane;
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if (r0 + u < end && ci < cpr) v = ld_nc_v4(X + (r0 + u) * cpr + ci);
        fma_chunk(v, qr[c], acc[u]);
      }
    }
    warp_transpose_reduce<4>(acc, lane);
    const int64_t my_r = r0 + (lane >> 3);
    if ((lane & 7) == 0 && my_r < end && acc[0] > thresh) range_append(out, cap, counter, acc[0], (uint32_t)my_r);
  }
}

typedef void (*ivf_range_fn)(const uint4*, int, const float*, const unsigned long long*, int, int, const int64_t*, float,
                             unsigned long long*, unsigned int, unsigned int*);
static ivf_range_fn pick_ivf_range(int ch) {
  switch (ch) {
    case 1: return ivf_range_kernel<1>;
    case 2: return ivf_range_kernel<2>;
    case 3: return ivf_range_kernel<3>;
    case 4: return ivf_range_kernel<4>;
    case 5: return ivf_range_kernel<5>;
    case 6: return ivf_range_kernel<6>;
    case 7: return ivf_range_kernel<7>;
    case 8: return ivf_range_kernel<8>;
  }
  return nullptr;
}

// One query (device pointer): (score, slot) keys of every probed row above `thresh`; *d_count = number of hits.
int ivf_range_scan(b200_index* idx, const float* d_q, float thresh, unsigned long long* d_out, unsigned int cap,
                   unsigned int* d_count, cudaStream_t st) {
  const int d = idx->d, cpr = d / 8, ch = (cpr + 31) / 32;
  const int nprobe = std::min(idx->nprobe, idx->nlist);
  void* ws = nullptr;
  B200_TRY(index_ws(idx, 3, (size_t)nprobe * 8, &ws));
  unsigned long long* probes = (unsigned long long*)ws;
  B200_TRY(scan_topk_keys(idx, idx->centroids, idx->nlist, d_q, 1, nprobe, probes, st));
  ivf_range_fn fn = pick_ivf_range(ch);
  B200_CHECK(fn != nullptr, B200_ERR_UNSUPPORTED, "ivf range_search: unsupported dimension %d", d);
  B200_CUDA(cudaMemsetAsync(d_count, 0, sizeof(unsigned int), st));
  const int segs = list_segments(idx, 2 * idx->sms, nprobe, 256);
  fn<<<(unsigned)(nprobe * segs), 256, 0, st>>>(reinterpret_cast<const uint4*>(idx->rows), cpr, d_q, probes, nprobe, segs,
                                                 idx->list_offsets, thresh, d_out, cap, d_count);
  B200_LAUNCH_OK();
  return B200_OK;
}

}  // namespace b200

// ---- k-means training of the coarse quantiser (SURVEY §8(f) row 2) -----------------------------------
// The GPU counterpart of the training step behind `clip-retrieval index` (clip_index.py:12-31 ->
// autofaiss.build_index -> faiss Clustering): Lloyd iterations under the index's own assignment rule
// (centroid of maximum inner product, ties to the lower list id, centroids rounded to fp16 exactly as
// b200_index_create_ivfflat stores them), centroid = mean of its rows, FAISS-style split of empty
// clusters.  Assignment reuses ivf_assign_kernel; the update is a deterministic segmented sum: rows
// are radix-sorted by list (stable, so ascending row id inside a list) and one CTA per list adds them
// in that order, thread = column — the same rows always give the same centroids.
namespace b200 {

__global__ void kmeans_gather_kernel(const __half* __restrict__ X, int d, const int64_t* __restrict__ pick, int nlist,
                                     float* __restrict__ C32) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)nlist * d) return;
  const int l = (int)(i / d), j = (int)(i - (int64_t)l * d);
  C32[i] = __half2float(X[pick[l] * d + j]);
}

__global__ void kmeans_to_half_kernel(const float* __restrict__ C32, int64_t count, __half* __restrict__ C16) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) C16[i] = __float2half_rn(C32[i]);
}

// block = list; thread = column (strided); rows of the list in ascending row id.
__global__ void __launch_bounds__(256)
kmeans_update_kernel(const __half* __restrict__ X, int d, const uint32_t* __restrict__ sorted_src,
                     const int64_t* __restrict__ offsets, float* __restrict__ C32, int spherical) {
  const int l = blockIdx.x;
  const int64_t p0 = offsets[l], p1 = offsets[l + 1];
  if (p1 == p0) return;   // empty: handled by the split step
  const float inv = 1.0f / (float)(p1 - p0);
  __shared__ float s_part[256];
  float n2 = 0.f;
  for (int j = threadIdx.x; j < d; j += blockDim.x) {
    float s = 0.f;
    for (int64_t p = p0; p < p1; p++) s += __half2float(X[(int64_t)sorted_src[p] * d + j]);
    const float m = s * inv;
    C32[(int64_t)l * d + j] = m;
    n2 = fmaf(m, m, n2);
  }
  if (!spherical) return;
  s_part[threadIdx.x] = n2;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) s_part[threadIdx.x] += s_part[threadIdx.x + o];
    __syncthreads();
  }
  const float nrm = sqrtf(s_part[0]);
  if (nrm > 0.f)
    for (int j = threadIdx.x; j < d; j += blockDim.x) C32[(int64_t)l * d + j] /= nrm;
}

// FAISS Clustering::split_clusters, made deterministic: the empty list `ci` takes the centroid of `cj`
// and the two are perturbed symmetrically (1 +- 1/1024, alternating by column).
__global__ void kmeans_split_kernel(float* __restrict__ C32, int d, int ci, int cj) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= d) return;
  const float eps = 1.0f / 1024.0f;
  const float v = C32[(int64_t)cj * d + j];
  if (j % 2 == 0) {
    C32[(int64_t)ci * d + j] = v * (1.0f + eps);
    C32[(int64_t)cj * d + j] = v * (1.0f - eps);
  } else {
    C32[(int64_t)ci * d + j] = v * (1.0f - eps);
    C32[(int64_t)cj * d + j] = v * (1.0f + eps);
  }
}

static inline uint64_t kmeans_mix(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

}  // namespace b200

extern "C" int b200_kmeans_train_f16(const void* d_rows, int64_t n, int d, int nlist, int niter, uint64_t seed,
                                     int spherical, float* h_centroids, int64_t* h_sizes, int device) {
  using namespace b200;
  B200_CHECK(d_rows && h_centroids, B200_ERR_INVALID, "kmeans_train: null argument");
  B200_CHECK(d >= 8 && d % 8 == 0 && d <= 2048, B200_ERR_INVALID, "kmeans_train: d=%d (multiple of 8, <= 2048)", d);
  B200_CHECK(nlist >= 1 && n >= nlist && n < (1ll << 31) && niter >= 0, B200_ERR_INVALID,
             "kmeans_train: n=%lld nlist=%d niter=%d (need nlist <= n < 2^31)", (long long)n, nlist, niter);
  DeviceGuard g(device);
  const __half* X = (const __half*)d_rows;
  const int cpr = d / 8;
  const size_t count = (size_t)nlist * d;
  float* C32 = nullptr; __half* C16 = nullptr; int64_t* d_pick = nullptr; int64_t* d_off = nullptr;
  uint32_t *assign = nullptr, *src = nullptr, *assign2 = nullptr, *src2 = nullptr;
  void* tmp = nullptr;
  std::vector<void*> frees;
  auto cleanup = [&]() { for (void* p : frees) cudaFree(p); };
  auto alloc = [&](void** p, size_t bytes) -> int {
    B200_CUDA(cudaMalloc(p, bytes));
    frees.push_back(*p);
    return B200_OK;
  };
  int rc = [&]() -> int {
    B200_TRY(alloc((void**)&C32, count * 4));
    B200_TRY(alloc((void**)&C16, count * 2));
    B200_TRY(alloc((void**)&d_pick, (size_t)nlist * 8));
    B200_TRY(alloc((void**)&d_off, (size_t)(nlist + 1) * 8));
    B200_TRY(alloc((void**)&assign, (size_t)n * 4));
    B200_TRY(alloc((void**)&src, (size_t)n * 4));
    B200_TRY(alloc((void**)&assign2, (size_t)n * 4));
    B200_TRY(alloc((void**)&src2, (size_t)n * 4));
    // initial centroids: one seeded pick inside each of nlist equal strides of the rows (all distinct)
    std::vector<int64_t> pick(nlist);
    for (int i = 0; i < nlist; i++) {
      const int64_t lo = (int64_t)(((__int128)i * n) / nlist), hi = (int64_t)(((__int128)(i + 1) * n) / nlist);
      const uint64_t span = (uint64_t)std::max<int64_t>(1, hi - lo);
      pick[i] = lo + (int64_t)(kmeans_mix(seed ^ ((uint64_t)i * 0xD1342543DE82EF95ull)) % span);
    }
    B200_CUDA(cudaMemcpy(d_pick, pick.data(), (size_t)nlist * 8, cudaMemcpyHostToDevice));
    kmeans_gather_kernel<<<(unsigned)((count + 255) / 256), 256>>>(X, d, d_pick, nlist, C32);
    B200_LAUNCH_OK();
    size_t tmp_bytes = 0;
    B200_TRY(sort_pairs_by_list(nullptr, tmp_bytes, assign, assign2, src, src2, n, nlist, d_off));
    B200_TRY(alloc(&tmp, tmp_bytes));
    ivf_assign_fn afn = pick_ivf_assign((cpr + 31) / 32);
    B200_CHECK(afn != nullptr, B200_ERR_UNSUPPORTED, "kmeans_train: d=%d", d);
    std::vector<int64_t> off(nlist + 1);
    for (int it = 0; it <= niter; it++) {
      // assignment under the fp16-rounded centroids (the rule the index itself applies on add)
      kmeans_to_half_kernel<<<(unsigned)((count + 255) / 256), 256>>>(C32, (int64_t)count, C16);
      B200_LAUNCH_OK();
      afn<<<(unsigned)((n + 7) / 8), 256>>>(reinterpret_cast<const uint4*>(X), n, cpr, reinterpret_cast<const uint4*>(C16),
                                            nlist, assign);
      B200_LAUNCH_OK();
      iota_kernel<<<(unsigned)((n + 255) / 256), 256>>>(src, n, 0u);
      B200_LAUNCH_OK();
      B200_TRY(sort_pairs_by_list(tmp, tmp_bytes, assign, assign2, src, src2, n, nlist, d_off));
      B200_CUDA(cudaMemcpy(off.data(), d_off, (size_t)(nlist + 1) * 8, cudaMemcpyDeviceToHost));
      if (it == niter) break;   // the last round only refreshes the sizes of the final centroids
      kmeans_update_kernel<<<nlist, 256>>>(X, d, src2, d_off, C32, spherical);
      B200_LAUNCH_OK();
      // empty clusters: split the (currently) largest one, ties to the lower id; sizes halve as in FAISS
      std::vector<int64_t> sz(nlist);
      for (int l = 0; l < nlist; l++) sz[l] = off[l + 1] - off[l];
      for (int ci = 0; ci < nlist; ci++) {
        if (sz[ci] != 0) continue;
        int cj = 0;
        for (int l = 1; l < nlist; l++)
          if (sz[l] > sz[cj]) cj = l;
        if (sz[cj] < 2) break;
        kmeans_split_kernel<<<(d + 255) / 256, 256>>>(C32, d, ci, cj);
        B200_LAUNCH_OK();
        sz[ci] = sz[cj] / 2;
        sz[cj] -= sz[ci];
      }
    }
    B200_CUDA(cudaMemcpy(h_centroids, C32, count * 4, cudaMemcpyDeviceToHost));
    if (h_sizes)
      for (int l = 0; l < nlist; l++) h_sizes[l] = off[l + 1] - off[l];
    return B200_OK;
  }();
  cudaDeviceSynchronize();
  cleanup();
  return rc;
}
