// Search path, IVF-PQ (8-bit codes, inner product): the index type autofaiss writes for large collections
// (OPQ{M}_{d},IVF{nlist}_HNSW32,PQ{M}x8), served from the codes themselves.  FAISS IndexIVFPQ semantics (DESIGN §5):
//   score(q, row in list l) = dis0(l) + sum_{m < M} T[m][code_m],   all fp32,
//   T[m][j] = sum_{t < dsub} q[m dsub + t] * codebook[m][j][t]       (one table per query: IP does not depend on l),
//   dis0(l) = q . centroid_l from the fp32 centroids when by_residual, else 0.
// Search = (0) optional pre-transform q' = A q + b; (1) coarse: fp32 FMA scores against every centroid, top nprobe
// (exact, where FAISS's HNSW quantiser is approximate); (2) the tables T; (3) list scan: the table of one query sits
// in shared memory, one thread scores one code row by lookups, rows enter the per-warp candidate lists of the
// IVF-Flat scan (keys by insertion id); when table + lists exceed one CTA's shared memory the M sub-quantisers
// are split over a thread-block cluster of 2 or 4 CTAs whose partial sums meet in the leader CTA through
// distributed shared memory; (4) the chunked bitonic select.
// Codes are stored list after list at a pitch of round_up(M, 16) bytes (zero padding), so the IVF-Flat finalize
// path buckets them as rows of row_bytes, and a row's code bytes load as whole 16-byte vectors.
#include "index.cuh"
#include "ptx.cuh"
#include "scan.cuh"
#include <float.h>
#include <algorithm>
#include <cmath>
#include <vector>

namespace b200 {

constexpr int PQ_KSUB = 256;
constexpr int PQ_THREADS = 256;                 // list-scan CTA: 8 warps at most, one code row per thread
constexpr size_t PQ_SMEM_BUDGET = 200 * 1024;   // shared memory one list-scan CTA may take

static int pq_pitch(int M) { return (M + 15) / 16 * 16; }

// ---- (0) pre-transform: one warp per (query, output column) -----------------------------------------
__global__ void pq_pretransform_kernel(const float* __restrict__ X, int nq, int d_in, const float* __restrict__ A,
                                       const float* __restrict__ b, int d, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t w = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w >= (int64_t)nq * d) return;
  const int q = (int)(w / d), i = (int)(w - (int64_t)q * d);
  const float* x = X + (int64_t)q * d_in;
  const float* a = A + (int64_t)i * d_in;
  float s = 0.f;
  for (int j = lane; j < d_in; j += 32) s = fmaf(a[j], x[j], s);
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(FULL, s, o);
  if (lane == 0) out[w] = b ? s + b[i] : s;
}

// ---- (1) coarse step: keys[q][l] = (q . c_l, l) in fp32, 64 x 64 tiles, 4 x 4 per thread ---------------
constexpr int CQ_T = 64, CQ_K = 16;
__global__ void __launch_bounds__(256)
pq_coarse_kernel(const float* __restrict__ Q, int nq, const float* __restrict__ Cn, int nlist, int d,
                 unsigned long long* __restrict__ keys) {
  __shared__ float sq[CQ_K][CQ_T + 1], sc[CQ_K][CQ_T + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int l0 = blockIdx.x * CQ_T, q0 = blockIdx.y * CQ_T;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < d; k0 += CQ_K) {
    for (int i = threadIdx.x; i < CQ_T * CQ_K; i += 256) {
      const int r = i / CQ_K, c = i % CQ_K;
      sq[c][r] = (q0 + r < nq && k0 + c < d) ? Q[(int64_t)(q0 + r) * d + k0 + c] : 0.f;
      sc[c][r] = (l0 + r < nlist && k0 + c < d) ? Cn[(int64_t)(l0 + r) * d + k0 + c] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int c = 0; c < CQ_K; c++) {
      float a[4], bb[4];
#pragma unroll
      for (int u = 0; u < 4; u++) { a[u] = sq[c][ty + 16 * u]; bb[u] = sc[c][tx + 16 * u]; }
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
      const int q = q0 + ty + 16 * u, l = l0 + tx + 16 * v;
      if (q < nq && l < nlist) keys[(int64_t)q * nlist + l] = make_key(acc[u][v], (uint32_t)l);
    }
}

// ---- (2) tables: T[q][m][j], m < pitch (rows M..pitch-1 are zero: they meet the zero padding of the codes) ----
__global__ void pq_tables_kernel(const float* __restrict__ Q, int d, int M, int dsub, const float* __restrict__ cb,
                                 float* __restrict__ T) {
  const int q = blockIdx.y, m = blockIdx.x, j = threadIdx.x;
  float s = 0.f;
  if (m < M) {
    const float* x = Q + (int64_t)q * d + m * dsub;
    const float* c = cb + ((int64_t)m * PQ_KSUB + j) * dsub;
    for (int t = 0; t < dsub; t++) s = fmaf(x[t], c[t], s);
  }
  T[((int64_t)q * gridDim.x + m) * PQ_KSUB + j] = s;
}

// ---- (3) list scan ------------------------------------------------------------------------------------
// Grid: clusters of `cs` CTAs; cluster c serves query c / cpq and takes work items (probe, segment)
// c % cpq, + cpq, ...  CTA `rank` of the cluster holds table rows [rank * mc, rank * mc + mc) of its query (loaded
// once per CTA) and scores those code bytes of every row; ranks > 0 store their partial sums into the leader's
// double-buffered exchange slots (one cluster barrier per pass of PQ_THREADS rows), the leader adds them, adds
// nothing else, and inserts.  The leader starts each row's sum at dis0, so with cs = 1 the fp32 sum runs
// dis0 + T[0] + T[1] + ... in m order.
// RANGE: no lists; every row scoring strictly above `thresh` is appended as a (score, slot) key.
// `codes` / `offsets` are the resident list store, or a staging arena of the lists a pass probes (lists in host
// memory, knn_ivfpq_stream.cu) whose probe keys name arena lists; row_ids == nullptr: a key's id is its row r.
template <bool RANGE>
__global__ void __launch_bounds__(PQ_THREADS)
ivfpq_scan_kernel(const uint8_t* __restrict__ codes, int pitch, const uint32_t* __restrict__ row_ids,
                  const float* __restrict__ tables, const unsigned long long* __restrict__ probes, int nprobe, int segs,
                  int cpq, const int64_t* __restrict__ offsets, int by_residual, int mc, int cs, int k,
                  unsigned long long* __restrict__ out_keys, int64_t out_stride_q, float thresh, unsigned int cap,
                  unsigned int* __restrict__ counter) {
  extern __shared__ __align__(16) unsigned char pq_smem[];
  float* s_tab = reinterpret_cast<float*>(pq_smem);                          // [mc][256]
  float* s_xchg = s_tab + (size_t)mc * PQ_KSUB;                               // [2][cs - 1][PQ_THREADS] (leader)
  unsigned long long* s_keys =
      reinterpret_cast<unsigned long long*>(s_xchg + (size_t)2 * (cs - 1) * PQ_THREADS);   // [warps][k]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nthreads = blockDim.x;
  const int rank = cs > 1 ? (int)ptx::cluster_ctarank() : 0;
  const int cluster = blockIdx.x / cs;
  const int q = cluster / cpq, g = cluster % cpq;
  const int m0 = min(rank * mc, pitch), m1 = min(m0 + mc, pitch);
  const float* tq = tables + ((int64_t)q * pitch + m0) * PQ_KSUB;
  for (int i = tid; i < (m1 - m0) * PQ_KSUB; i += nthreads) s_tab[i] = tq[i];
  unsigned long long* wkeys = s_keys + (size_t)warp * k;
  if (!RANGE) warp_lists_clear(wkeys, k, lane);
  if (cs > 1) ptx::cluster_sync();   // every CTA of the cluster runs before the first remote store
  else __syncthreads();
  const uint32_t xchg_remote = cs > 1 ? ptx::mapa_shared(ptx::smem_u32(s_xchg), 0) : 0u;
  unsigned long long worst = 0ull;
  int worst_pos = 0, par = 0;
  const int nvec = (m1 - m0) / 16;
  for (int item = g; item < nprobe * segs; item += cpq) {
    const int p = item / segs, seg = item % segs;
    const unsigned long long pk = probes[(int64_t)q * nprobe + p];
    if (pk == 0ull) continue;   // uniform over the cluster: same query, same item
    const float dis0 = by_residual ? key_score(pk) : 0.f;
    int64_t beg, end;
    segment_rows(offsets, key_id(pk), segs, seg, 1, beg, end);
    for (int64_t r0 = beg; r0 < end; r0 += nthreads) {
      const int64_t r = r0 + tid;
      const bool live = r < end;
      float s = rank == 0 ? dis0 : 0.f;
      if (live) {
        const uint4* src = reinterpret_cast<const uint4*>(codes + r * pitch + m0);
        for (int c = 0; c < nvec; c++) {
          const uint4 v = __ldg(src + c);
          const uint32_t w4[4] = {v.x, v.y, v.z, v.w};
          const float* t = s_tab + (size_t)c * 16 * PQ_KSUB;
#pragma unroll
          for (int b = 0; b < 16; b++) s += t[b * PQ_KSUB + ((w4[b >> 2] >> ((b & 3) * 8)) & 0xffu)];
        }
      }
      if (cs > 1) {
        if (rank > 0)
          ptx::st_shared_cluster_f32(xchg_remote + (uint32_t)(((par * (cs - 1) + rank - 1) * PQ_THREADS + tid) * 4), s);
        ptx::cluster_sync();
        if (rank == 0)
          for (int rr = 1; rr < cs; rr++) s += s_xchg[(par * (cs - 1) + rr - 1) * PQ_THREADS + tid];
        par ^= 1;
      }
      if (rank != 0) continue;
      if (RANGE) {
        if (live && s > thresh) range_append(out_keys, cap, counter, s, (uint32_t)r);
        continue;
      }
      // Only a row scoring at least the worst kept score can enter the list (as in the IVF-Flat scan).
      const bool reach = live && (s == s) && f32_to_ordered(s) >= (uint32_t)(worst >> 32);
      unsigned long long key = 0ull;
      if (reach) key = make_key(s, row_ids ? __ldg(row_ids + r) : (uint32_t)r);
      warp_offer(wkeys, k, reach && key > worst, key, &worst, &worst_pos, lane);
    }
  }
  if (RANGE || rank != 0) return;
  __syncwarp();
  warp_list_store(out_keys + (int64_t)q * out_stride_q + ((int64_t)g * (nthreads >> 5) + warp) * k, wkeys, k, lane);
}

// ---- (4) decode: rows for keys (search_and_reconstruct) or ids (reconstruct) ----------------------------
// One warp per row: y[j] = codebook[m][code_m][t] + centroid_l[j] (fp32 add; no centroid without residuals), then
// x = A^T (y - b) when a pre-transform is set.  Key 0 / an id outside the shard -> all-ones bits (NaN).
// A staging arena decodes with id_to_slot == nullptr (a key's id is its arena row) and `list_ids` mapping an arena
// list to the index's list, whose centroid the row adds; the resident store passes list_ids == nullptr.
__global__ void pq_decode_kernel(const uint8_t* __restrict__ codes, int pitch, int M, int dsub, int d,
                                 const float* __restrict__ cb, const float* __restrict__ cent, int by_residual,
                                 const int64_t* __restrict__ offsets, int nlist, const int32_t* __restrict__ list_ids,
                                 const uint32_t* __restrict__ id_to_slot,
                                 const unsigned long long* __restrict__ keys, const int64_t* __restrict__ ids,
                                 int64_t id_base, int64_t ntotal, int64_t count, const float* __restrict__ A,
                                 const float* __restrict__ b, int d_in, float* __restrict__ out) {
  extern __shared__ float s_y[];   // [warps][d] when A is set
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t w = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
  if (w >= count) return;
  float* o = out + w * d_in;
  int64_t local = -1;
  if (keys) {
    if (keys[w] != 0ull) local = key_id(keys[w]);
  } else if (ids[w] >= 0 && ids[w] - id_base >= 0 && ids[w] - id_base < ntotal) {
    local = ids[w] - id_base;
  }
  if (local < 0) {
    for (int j = lane; j < d_in; j += 32) o[j] = __uint_as_float(0xffffffffu);
    return;
  }
  const int64_t slot = id_to_slot ? (int64_t)id_to_slot[local] : local;
  int lo = 0, hi = nlist;   // list of the slot: offsets[l] <= slot < offsets[l + 1]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (offsets[mid] <= slot) lo = mid; else hi = mid;
  }
  const uint8_t* row = codes + slot * pitch;
  float* y = A ? s_y + (size_t)warp * d : o;
  for (int j = lane; j < d; j += 32) {
    const int m = j / dsub, t = j - m * dsub;
    const float c = cb[((int64_t)m * PQ_KSUB + row[m]) * dsub + t];
    y[j] = by_residual ? __fadd_rn(c, cent[(int64_t)(list_ids ? list_ids[lo] : lo) * d + j]) : c;
  }
  if (!A) return;
  __syncwarp();
  for (int i = lane; i < d_in; i += 32) {
    float s = 0.f;
    for (int j = 0; j < d; j++) s = fmaf(A[(int64_t)j * d_in + i], b ? y[j] - b[j] : y[j], s);
    o[i] = s;
  }
}

// ---- host side ------------------------------------------------------------------------------------------

// The smallest cluster (1, 2, 4 CTAs) whose share of the table plus candidate lists leaves at least 4 warps of
// lists in the budget; failing that, the most warps.  Depends on (M, k) alone, so every query batch of a shape
// sums its rows in the same order.
static PqPlan pq_plan(int pitch, int k) {
  PqPlan best;
  for (int cs = 1; cs <= 4; cs <<= 1) {
    const int mc = ((pitch + cs - 1) / cs + 15) / 16 * 16;
    for (int w = PQ_THREADS / 32; w >= 1; w >>= 1) {
      const size_t smem = (size_t)mc * PQ_KSUB * 4 + (size_t)2 * (cs - 1) * PQ_THREADS * 4 + (size_t)w * k * 8;
      if (smem <= PQ_SMEM_BUDGET) {
        if (w > best.warps) best = PqPlan{cs, mc, w, smem};
        break;
      }
    }
    if (best.warps >= 4) break;
  }
  return best;
}

static int pq_launch_scan(b200_index* idx, const PqSearch& s, const PqStore& store, bool range, int nq,
                          const float* tables, const unsigned long long* probes, unsigned long long* out, float thresh,
                          unsigned int cap, unsigned int* counter, cudaStream_t st) {
  const PqPlan& pl = s.pl;
  const void* fn = range ? (const void*)ivfpq_scan_kernel<true> : (const void*)ivfpq_scan_kernel<false>;
  if (pl.smem > 48 * 1024) B200_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)((int64_t)nq * s.cpq * pl.cs));
  cfg.blockDim = dim3(range ? PQ_THREADS : pl.warps * 32);
  cfg.dynamicSmemBytes = pl.smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = pl.cs;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pl.cs > 1 ? 1 : 0;
  const int pitch = idx->row_bytes, by_res = idx->pq_by_residual ? 1 : 0;
  if (range)
    B200_CUDA(cudaLaunchKernelEx(&cfg, ivfpq_scan_kernel<true>, store.codes, pitch, store.row_ids, tables, probes, s.nprobe,
                                 s.segs, s.cpq, store.offsets, by_res, pl.mc, pl.cs, s.k, out, s.Mq, thresh, cap, counter));
  else
    B200_CUDA(cudaLaunchKernelEx(&cfg, ivfpq_scan_kernel<false>, store.codes, pitch, store.row_ids, tables, probes, s.nprobe,
                                 s.segs, s.cpq, store.offsets, by_res, pl.mc, pl.cs, s.k, out, s.Mq, thresh, cap, counter));
  B200_LAUNCH_OK();
  return B200_OK;
}

int pq_search_plan(b200_index* idx, int nq, int k, PqSearch* s) {
  s->nprobe = std::min(idx->nprobe, idx->nlist);
  s->k = k;
  // select plan of the coarse step: k = nprobe over the nlist scores of a query (two select levels, as the list scan)
  B200_CHECK((size_t)select_buffer(s->nprobe) * 8 <= SELECT_SMEM_MAX, B200_ERR_UNSUPPORTED,
             "ivfpq %s: nprobe=%d exceeds the supported maximum (12800)", k ? "search" : "range_search", s->nprobe);
  B200_TRY(plan_select(idx->nlist, s->nprobe, &s->cp));
  s->pl = pq_plan(idx->row_bytes, k);
  B200_CHECK(s->pl.warps >= 1, B200_ERR_UNSUPPORTED, "search: k=%d exceeds the supported maximum (8192)", k);
  s->qmax = std::min(PQ_QB, nq);
  // clusters per query: enough to fill the chip twice; segments of at least ~PQ_THREADS rows
  const int target = std::max(1, 2 * idx->sms / s->pl.cs);
  s->segs = list_segments(idx, target, (int64_t)s->qmax * s->nprobe, PQ_THREADS);
  s->cpq = (int)std::min<int64_t>((int64_t)s->nprobe * s->segs, std::max<int64_t>(1, (target + s->qmax - 1) / s->qmax));
  s->Mq = (int64_t)s->cpq * s->pl.warps * k;   // candidates per query
  B200_TRY(plan_select(s->Mq, k, &s->sel));
  const size_t w4 = ((((size_t)s->qmax * idx->d + 63) & ~(size_t)63) + (size_t)s->qmax * idx->row_bytes * PQ_KSUB) * 4;
  B200_TRY(index_ws(idx, 0, std::max(s->cp.keys(s->qmax), s->sel.keys(s->qmax)) * 8, (void**)&s->w0));
  B200_TRY(index_ws(idx, 3, (size_t)s->qmax * s->nprobe * 8, (void**)&s->probes));
  return index_ws(idx, 4, w4, (void**)&s->w4);
}

int pq_prepare(b200_index* idx, const PqSearch& s, const float* d_q, int qb, bool probes, float** tables, cudaStream_t st) {
  const int d = idx->d, nlist = idx->nlist;
  const float* q = d_q;
  float* t = s.w4;
  if (idx->pt_A) {   // (0) q' = A q + b at the start of w4, the tables after it
    t = s.w4 + (((size_t)qb * d + 63) & ~(size_t)63);
    const int64_t warps = (int64_t)qb * d;
    pq_pretransform_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, st>>>(d_q, qb, idx->d_in, idx->pt_A, idx->pt_b, d, s.w4);
    B200_LAUNCH_OK();
    q = s.w4;
  }
  if (probes) {   // (1) probe keys: fp32 coarse score = dis0, list id
    pq_coarse_kernel<<<dim3((nlist + CQ_T - 1) / CQ_T, (qb + CQ_T - 1) / CQ_T), 256, 0, st>>>(q, qb, idx->pq_centroids,
                                                                                            nlist, d, s.w0);
    B200_LAUNCH_OK();
    B200_TRY(select_topk(s.cp, s.w0, s.w0 + (size_t)qb * nlist, s.probes, qb, st));
  }
  if (!tables) return B200_OK;
  *tables = t;   // (2)
  pq_tables_kernel<<<dim3(idx->row_bytes, qb), PQ_KSUB, 0, st>>>(q, d, idx->pq_M, d / idx->pq_M, idx->pq_codebook, t);
  B200_LAUNCH_OK();
  return B200_OK;
}

int pq_scan_select(b200_index* idx, const PqSearch& s, const PqStore& store, int qb, const float* tables,
                   const unsigned long long* probes, unsigned long long* out, cudaStream_t st) {
  B200_TRY(scan_timer_begin(idx, st));
  B200_TRY(pq_launch_scan(idx, s, store, false, qb, tables, probes, s.w0, 0.f, 0, nullptr, st));
  B200_TRY(scan_timer_end(idx, st));
  idx->last_scan_launches++;
  B200_TRY(select_topk(s.sel, s.w0, s.w0 + (size_t)qb * s.Mq, out, qb, st));
  idx->last_scan_plan[0] = 4;
  idx->last_scan_plan[1] = s.pl.mc;
  idx->last_scan_plan[2] = s.pl.cs;
  idx->last_scan_plan[3] = s.pl.warps;
  return B200_OK;
}

int pq_scan_range(b200_index* idx, const PqSearch& s, const PqStore& store, const float* tables,
                  const unsigned long long* probes, float thresh, unsigned long long* out, unsigned int cap,
                  unsigned int* counter, cudaStream_t st) {
  B200_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned int), st));
  return pq_launch_scan(idx, s, store, true, 1, tables, probes, out, thresh, cap, counter, st);
}

static PqStore resident_store(const b200_index* idx) {
  return PqStore{reinterpret_cast<const uint8_t*>(idx->rows), idx->row_ids, idx->list_offsets};
}

int ivfpq_search_keys(b200_index* idx, const float* d_q, int nq, int k, unsigned long long* d_keys, cudaStream_t st) {
  PqSearch s;
  B200_TRY(pq_search_plan(idx, nq, k, &s));
  idx->ev_used = 0;
  for (int q0 = 0; q0 < nq; q0 += PQ_QB) {
    const int qb = std::min(PQ_QB, nq - q0);
    float* tables = nullptr;
    B200_TRY(pq_prepare(idx, s, d_q + (size_t)q0 * idx->d_in, qb, true, &tables, st));
    B200_TRY(pq_scan_select(idx, s, resident_store(idx), qb, tables, s.probes, d_keys + (size_t)q0 * k, st));
  }
  return B200_OK;
}

// One query (device pointer): (score, slot) keys of every row of the probed lists scoring strictly above `thresh`.
int ivfpq_range_scan(b200_index* idx, const float* d_q, float thresh, unsigned long long* d_out, unsigned int cap,
                     unsigned int* d_count, cudaStream_t st) {
  PqSearch s;
  B200_TRY(pq_search_plan(idx, 1, 0, &s));
  float* tables = nullptr;
  B200_TRY(pq_prepare(idx, s, d_q, 1, true, &tables, st));
  return pq_scan_range(idx, s, resident_store(idx), tables, s.probes, thresh, d_out, cap, d_count, st);
}

int ivfpq_decode(b200_index* idx, const unsigned long long* keys, const int64_t* ids, int64_t count, float* d_R,
                 cudaStream_t st) {
  return pq_decode_launch(idx, reinterpret_cast<const uint8_t*>(idx->rows), idx->list_offsets, idx->nlist, nullptr,
                          idx->id_to_slot, keys, ids, count, d_R, st);
}

int pq_decode_launch(b200_index* idx, const uint8_t* codes, const int64_t* offsets, int nlists, const int32_t* list_ids,
                     const uint32_t* id_to_slot, const unsigned long long* keys, const int64_t* ids, int64_t count,
                     float* d_R, cudaStream_t st) {
  if (count == 0) return B200_OK;
  const int warps = 4;
  const size_t smem = idx->pt_A ? (size_t)warps * idx->d * 4 : 0;
  pq_decode_kernel<<<(unsigned)((count + warps - 1) / warps), warps * 32, smem, st>>>(
      codes, idx->row_bytes, idx->pq_M, idx->d / idx->pq_M, idx->d, idx->pq_codebook, idx->pq_centroids,
      idx->pq_by_residual ? 1 : 0, offsets, nlists, list_ids, id_to_slot, keys, ids, idx->id_base, idx->ntotal, count,
      idx->pt_A, idx->pt_b, idx->d_in, d_R);
  B200_LAUNCH_OK();
  return B200_OK;
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_index_create_ivfpq(int d, int nlist, int M, int by_residual, const float* h_centroids, const float* h_codebook,
                            int device, b200_index** out) {
  B200_CHECK(nlist >= 1 && h_centroids != nullptr && h_codebook != nullptr, B200_ERR_INVALID,
             "create_ivfpq: bad nlist/centroids/codebook");
  B200_CHECK(M >= 1 && M <= 256 && d > 0 && d % M == 0, B200_ERR_INVALID,
             "create_ivfpq: M=%d must be in [1, 256] and divide d=%d", M, d);
  B200_TRY(b200_index_create_flat(d, device, out));
  b200_index* idx = *out;
  DeviceGuard g(device);
  auto init = [&]() -> int {
    B200_TRY(ivf_create(idx, nlist, nullptr));
    idx->pq_M = M;
    idx->pq_by_residual = by_residual != 0;
    idx->row_bytes = pq_pitch(M);
    const size_t nc = (size_t)nlist * d, nb = (size_t)PQ_KSUB * d;   // codebook: M * 256 * (d / M)
    B200_CUDA(cudaMalloc((void**)&idx->pq_centroids, nc * 4));
    B200_CUDA(cudaMemcpy(idx->pq_centroids, h_centroids, nc * 4, cudaMemcpyHostToDevice));
    B200_CUDA(cudaMalloc((void**)&idx->pq_codebook, nb * 4));
    B200_CUDA(cudaMemcpy(idx->pq_codebook, h_codebook, nb * 4, cudaMemcpyHostToDevice));
    return B200_OK;
  };
  const int rc = init();
  if (rc != B200_OK) {
    b200_index_destroy(idx);
    *out = nullptr;
  }
  return rc;
}

int b200_index_add_codes(b200_index* idx, const uint8_t* codes, int64_t n, int codes_on_device, const int32_t* h_lists) {
  B200_CHECK(idx && n >= 0 && (n == 0 || (codes && h_lists)), B200_ERR_INVALID, "add_codes: bad argument");
  B200_CHECK(idx->pq_M > 0, B200_ERR_STATE, "add_codes: not an IVF-PQ index");
  B200_CHECK(!idx->host, B200_ERR_STATE, "add_codes: the index serves lists in host memory (b200_index_set_host_lists)");
  for (int64_t i = 0; i < n; i++)
    B200_CHECK(h_lists[i] >= 0 && h_lists[i] < idx->nlist, B200_ERR_INVALID, "add_codes: row %lld has list %d of %d",
               (long long)i, h_lists[i], idx->nlist);
  if (n == 0) return B200_OK;
  B200_CHECK(idx->ntotal + idx->npending + n < (1ll << 32), B200_ERR_UNSUPPORTED, "add_codes: a shard holds at most 2^32 rows");
  idx->graph_epoch++;
  DeviceGuard g(idx->device);
  const int64_t rb = idx->row_bytes;
  B200_TRY(grow_pending(idx, idx->npending + n, true));
  uint8_t* dst = reinterpret_cast<uint8_t*>(idx->pending) + idx->npending * rb;
  if (rb != idx->pq_M) B200_CUDA(cudaMemset(dst, 0, (size_t)n * rb));   // the padding scores as the zero table rows
  B200_CUDA(cudaMemcpy2D(dst, (size_t)rb, codes, (size_t)idx->pq_M, (size_t)idx->pq_M, (size_t)n,
                         codes_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
  idx->pending_lists.resize((size_t)idx->npending, 0xFFFFFFFFu);
  for (int64_t i = 0; i < n; i++) idx->pending_lists.push_back((uint32_t)h_lists[i]);
  idx->npending += n;
  return B200_OK;
}

// FAISS LinearTransform::set_is_orthonormal: A A^T = I within 4e-5 (only when d_out <= d_in).
int b200_index_set_pretransform(b200_index* idx, int d_in, const float* h_A, const float* h_b) {
  B200_CHECK(idx && h_A, B200_ERR_INVALID, "set_pretransform: bad argument");
  B200_CHECK(idx->pq_M > 0, B200_ERR_STATE, "set_pretransform: not an IVF-PQ index");
  B200_CHECK(d_in >= 1 && d_in <= 2048, B200_ERR_INVALID, "set_pretransform: d_in=%d must be in [1, 2048]", d_in);
  const int d = idx->d;
  bool ortho = d <= d_in;
  for (int i = 0; i < d && ortho; i++)
    for (int j = 0; j < d && ortho; j++) {
      double s = 0;
      for (int t = 0; t < d_in; t++) s += (double)h_A[(size_t)i * d_in + t] * h_A[(size_t)j * d_in + t];
      if (std::fabs(s - (i == j ? 1.0 : 0.0)) > 4e-5) ortho = false;
    }
  DeviceGuard g(idx->device);
  std::lock_guard<std::mutex> lock(idx->mu);
  if (idx->pt_A) B200_CUDA(cudaFree(idx->pt_A));
  if (idx->pt_b) B200_CUDA(cudaFree(idx->pt_b));
  idx->pt_A = nullptr;
  idx->pt_b = nullptr;
  B200_CUDA(cudaMalloc((void**)&idx->pt_A, (size_t)d * d_in * 4));
  B200_CUDA(cudaMemcpy(idx->pt_A, h_A, (size_t)d * d_in * 4, cudaMemcpyHostToDevice));
  if (h_b) {
    B200_CUDA(cudaMalloc((void**)&idx->pt_b, (size_t)d * 4));
    B200_CUDA(cudaMemcpy(idx->pt_b, h_b, (size_t)d * 4, cudaMemcpyHostToDevice));
  }
  idx->d_in = d_in;
  idx->pt_orthonormal = ortho;
  idx->graph_epoch++;
  return B200_OK;
}

}  // extern "C"
