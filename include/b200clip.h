/*
 * b200clip.h — C ABI of the CUDA-native hot path (H100, sm_90a) for rom1504/clip-retrieval.
 *
 * The reference (pure Python) has no FFI of its own; its hot-path seams are duck-typed Python
 * objects (SURVEY.md §8b).  Each entry point below names the reference call it replaces.
 * Conventions:
 *   - every function returns 0 on success, a negative b200_status on failure; the message of the
 *     last failure on the calling thread is b200_last_error().  No exception crosses this ABI.
 *   - `h_` pointers are host memory, `d_` pointers are device memory on the handle's device.
 *   - `stream` is a cudaStream_t passed as void* (NULL = the legacy default stream).  Device entry
 *     points are asynchronous on `stream`; host entry points return after the result is in the
 *     host buffers.
 *   - the caller owns every buffer it passes in; the library owns what is behind the handles.
 *   - a handle may be searched / encoded concurrently from several threads only through the host
 *     entry points (they serialise on an internal mutex); `add`, `load`, `set_nprobe` are not
 *     concurrent-safe with anything.
 */
#ifndef B200CLIP_H
#define B200CLIP_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum b200_status {
  B200_OK = 0,
  B200_ERR_INVALID = -1,   /* bad argument */
  B200_ERR_CUDA = -2,      /* a CUDA runtime / driver call failed */
  B200_ERR_OOM = -3,       /* device allocation failed */
  B200_ERR_STATE = -4,     /* handle not in a state that allows the call */
  B200_ERR_UNSUPPORTED = -5
} b200_status;

const char* b200_last_error(void);
/* Library version string and the SM architecture it was compiled for ("sm_90a"). */
const char* b200_version(void);
/* Number of kernel launches this library has issued in this process (all handles, all streams).
 * bench.py reads it before/after the timed region to report `gpu_launches`. */
int64_t b200_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * Synthetic data (BASELINE.json configs are synthetic).  Counter-based and exactly reproducible
 * on the CPU (oracle/synth_ref.py): integer noise, integer sum of squares, one fp64 sqrt/divide.
 *   row r, col j:  noise(r,j) = sum of the 4 low bytes of splitmix64(seed, r, j) - 510
 *   mode 0 (iid):        v = noise
 *   mode 1 (clustered):  v = 8*noise(seed_c, list(r), j) + noise_scale_x8... see synth.cu
 *   x = v / sqrt(sum v^2)  (fp64) -> fp32 -> fp16
 * ------------------------------------------------------------------------------------------ */
typedef struct b200_synth_spec {
  uint64_t seed;          /* noise seed */
  int32_t  clustered;     /* 0: iid rows; 1: centroid[list(row)] * cw + noise * nw */
  uint64_t centroid_seed; /* clustered: seed of the centroid rows */
  int32_t  nlist;         /* clustered: number of centroids; list(row) = hash(row) % nlist */
  int32_t  cw, nw;        /* clustered: integer weights of centroid and noise */
} b200_synth_spec;

/* Fill `d_out` ([n, d] row-major) with rows row0 .. row0+n-1 of the synthetic set. */
int b200_synth_rows_f16(void* d_out, int64_t n, int d, int64_t row0, const b200_synth_spec* spec, void* stream);
int b200_synth_rows_f32(float* d_out, int64_t n, int d, int64_t row0, const b200_synth_spec* spec, void* stream);

/* ------------------------------------------------------------------------------------------
 * Search path.  Replaces the FAISS index object held in ClipResource.image_index/text_index
 * (reference clip_retrieval/clip_back.py:781-782), created by load_index (clip_back.py:589-596)
 * and queried by KnnService.knn_search through index.search_and_reconstruct(query, k)
 * (clip_back.py:362); secondary call sites index.search (clip_filter.py:55).
 * Metric: inner product (cosine on normalised rows), fp16 storage, fp32 accumulation.
 * Result order: score descending, ties by ascending id.  Unfilled slots: id -1, score -FLT_MAX,
 * reconstructed row all-ones bits (NaN) — what FAISS returns and clip_back.py:370-378 truncates.
 * ------------------------------------------------------------------------------------------ */
typedef struct b200_index b200_index;

/* Flat (exhaustive) index of dimension d (multiple of 8, <= 2048) on CUDA device `device`. */
int b200_index_create_flat(int d, int device, b200_index** out);
/* IVF-Flat: `h_centroids` is [nlist, d] fp32 on the host (rounded to fp16 inside, as the stored
 * rows are).  Rows are assigned to the centroid of maximum inner product (FAISS IVF, IP metric). */
int b200_index_create_ivfflat(int d, int nlist, const float* h_centroids, int device, b200_index** out);
/* IVF-PQ with 8-bit codes (FAISS IndexIVFPQ, inner product): `h_centroids` [nlist, d] fp32 (kept in fp32: they give
 * dis0), `h_codebook` [M, 256, d / M] fp32; 1 <= M <= 256, M divides d.  by_residual: score = q.c_l + ADC(codes), else
 * ADC(codes) alone.  Rows enter as codes through b200_index_add_codes; b200_index_encode_device makes those codes
 * (and lists) from float rows. */
int b200_index_create_ivfpq(int d, int nlist, int M, int by_residual, const float* h_centroids,
                            const float* h_codebook, int device, b200_index** out);
/* IVF-PQ only: append n code rows ([n, M] uint8) with their inverted lists (h_lists[i] in [0, nlist)); insertion ids
 * continue from ntotal. */
int b200_index_add_codes(b200_index* idx, const uint8_t* codes, int64_t n, int codes_on_device, const int32_t* h_lists);
/* IVF-PQ only: queries are d_in wide and searched as q' = A q (+ b), A [d, d_in] fp32 row-major, b [d] or NULL (FAISS
 * IndexPreTransform with one LinearTransform: an OPQ matrix or a random rotation).  Reconstruction returns
 * A^T (y - b), which needs orthonormal rows of A (checked here within 4e-5, as FAISS does); otherwise reconstruct and
 * search with rows return B200_ERR_UNSUPPORTED while search itself works.  b200_index_d reports d_in afterwards. */
int b200_index_set_pretransform(b200_index* idx, int d_in, const float* h_A, const float* h_b);
/* IVF-PQ only, on an index holding no rows: serve the lists from HOST memory (an on-disk index's memory map) instead
 * of HBM.  List l has h_sizes[l] rows; its M-byte code rows start at address h_code_addr[l] and its int64 ids at
 * h_id_addr[l].  The memory must stay mapped, unchanged, for the life of the handle; nothing is copied here.
 * Centroids, codebook and pre-transform stay on the device.  Each search pass copies the probes to the host, gathers
 * the probed lists (ascending list id, file order inside a list) into pinned staging, copies them to a device arena on
 * a copy stream and scans them there; two arenas overlap the gather and copy of one pass with the scan of the one
 * before.  Search, search_device, range_search, ivf_lists and ntotal keep their contracts; ids are the lists' own
 * (+ id_base), equal scores rank in list-order slot as in a resident load of the same lists, and every result equals
 * that resident load's bit for bit.  Searches are never captured in CUDA graphs and return with the stream
 * synchronised; reconstruct, add_codes and copy_rows return an error.  May be called again to re-point the lists. */
int b200_index_set_host_lists(b200_index* idx, int nlist, const int64_t* h_sizes, const uint64_t* h_code_addr,
                              const uint64_t* h_id_addr);
/* Lists in host memory: bytes per device arena (two are allocated, plus as much pinned staging).  An arena is never
 * smaller than nprobe x the largest list, so one query always fits; 0 = that least size.  Default 256 MiB. */
int b200_index_set_stream_arena(b200_index* idx, size_t bytes);
/* Lists in host memory, the last search or range_search: h_stats[4] = {host gather ms, copy ms (device events around
 * each pass's host-to-device copies), code bytes staged, passes}. */
int b200_index_last_stream_stats(const b200_index* idx, double* h_stats);
/* M of an IVF-PQ index; 0 for the other kinds. */
int b200_index_pq_m(const b200_index* idx);
/* IVF-PQ only: encode n fp32 rows d_x [n, width] (width = d_in when a pre-transform is set, else d; 16-byte aligned
 * without a pre-transform) on `stream`, asynchronously.  x' = A x + b (or x); d_lists [n] = argmax_l x'.c_l over the
 * fp32 centroids, ties to the lower list; d_residuals [n, d] = x' - c_list in fp32 (x' without by_residual);
 * d_codes [n, M] (unpadded) = per sub-quantiser the codeword of least fp32 sum of squared differences, ties to the
 * lower index.  Each output may be NULL.  Rows go through in chunks, so the scratch is bounded whatever n is.
 * `b200_index_add_codes(idx, codes, n, 1, lists)` then appends the rows. */
int b200_index_encode_device(b200_index* idx, const float* d_x, int64_t n, int32_t* d_lists, float* d_residuals,
                             uint8_t* d_codes, void* stream);
/* PQ training: M independent Lloyd k-means of 256 codewords (squared L2) on the sub-vectors of d_x [n, d] fp32 (device).
 * Initial codewords: one seeded pick per stride of the rows (as b200_kmeans_train_f16), the same for every m; each
 * codeword = mean of its rows added in ascending row order in fp32; an empty codeword takes a perturbed copy of the
 * largest one of the same m.  h_codebook [M, 256, d / M] fp32, h_sizes [M, 256] rows per codeword under the result
 * (or NULL).  Needs n >= 256, M dividing d, M * n < 2^31. */
int b200_pq_train_f32(const float* d_x, int64_t n, int d, int M, int niter, uint64_t seed, float* h_codebook,
                      int64_t* h_sizes, int device);
/* OPQ training (FAISS OPQMatrix::train, DESIGN §5 (xiii)): a rotation h_A [d_out, d_in] fp32 with orthonormal rows
 * (d_out <= d_in, M divides d_out) for the rows d_x [n, d_in] fp32 (device, 256 <= n <= 65536).  The start is the polar
 * factor of a seeded Gaussian matrix; each of `niter` iterations trains the PQ on the rotated rows (niter_pq_0 Lloyd
 * iterations from b200_pq_train_f32's seeded picks the first time, then niter_pq from the previous codebook), records
 * |x A^T - decode(codes)|^2 / n in h_objective[it] (or NULL), and sets A to the polar factor U V^T of
 * G = decode(codes)^T X (fp64 SVD).  The SVD is cuSOLVER's, resolved at run time: without libcusolver.so.11 the call
 * returns B200_ERR_UNSUPPORTED.  Deterministic: the same bits on every run.  h_phase_ms[4] (or NULL: no extra
 * synchronisation) receives the milliseconds spent in {rotating the rows, PQ training and objective, cross matrix,
 * SVD and polar product (the initial rotation included)}, measured between device synchronisations. */
int b200_opq_train_f32(const float* d_x, int64_t n, int d_in, int d_out, int M, int niter, int niter_pq, int niter_pq_0,
                       uint64_t seed, float* h_A, float* h_objective, float* h_phase_ms, int device);
/* The cross-matrix step of OPQ training alone: d_G [d_out, d_in] fp32 = Y^T X over the n <= 65536 rows, Y = the rows d_codes
 * [n, M] decode to under d_codebook [M, 256, d_out / M].  fp32 fma over fixed chunks of 1024 rows (ascending rows within
 * a chunk), the chunk partials added in chunk order. */
int b200_opq_cross_f32_device(const float* d_x, int64_t n, int d_in, const uint8_t* d_codes, const float* d_codebook,
                              int d_out, int M, float* d_G, int device, void* stream);
/* Rows d_y [n, d_out] = d_x [n, d_in] A^T (+ b), all fp32 on the device (A [d_out, d_in], b [d_out] or NULL), by the
 * kernel b200_index_encode_device pre-transforms with; d_y is fp32, or fp16 (rounded to nearest) with out_fp16. */
int b200_rows_pretransform_device(const float* d_x, int64_t n, int d_in, const float* d_A, const float* d_b, int d_out,
                                  void* d_y, int out_fp16, int device, void* stream);
/* The polar step alone: d_A [d_out, d_in] fp32 = U V^T for d_G = U S V^T [d_out, d_in] fp32 (d_out <= d_in), from the
 * fp64 SVD.  Synchronises the stream. */
int b200_opq_polar_f32_device(const float* d_G, int d_out, int d_in, float* d_A, int device, void* stream);
int b200_index_destroy(b200_index* idx);

/* Pre-size the row store (rows); avoids regrowth copies for large shards. */
int b200_index_reserve(b200_index* idx, int64_t n);
/* Append n rows ([n, d] row-major).  Ids are insertion positions + id_base (see set_id_base). */
int b200_index_add_f16(b200_index* idx, const void* rows, int64_t n, int rows_on_device);
int b200_index_add_f32(b200_index* idx, const float* rows, int64_t n, int rows_on_device);
/* IVF only: append n fp16 rows with an EXPLICIT inverted list per row (h_lists[i] in [0, nlist)) instead of the
 * max-inner-product assignment — how an existing FAISS IVF index file's own lists are kept (load_index,
 * clip_back.py:589-596). */
int b200_index_add_assigned_f16(b200_index* idx, const void* rows, int64_t n, int rows_on_device, const int32_t* h_lists);
/* Append n synthetic rows (rows row0.. of `spec`) generated directly in the row store. */
int b200_index_add_synthetic(b200_index* idx, int64_t n, int64_t row0, const b200_synth_spec* spec);
/* IVF only: rows appended since the last call are bucketed into their inverted lists.  Called
 * implicitly by the first search after an add. */
int b200_index_finalize(b200_index* idx);

int64_t b200_index_ntotal(const b200_index* idx);
int     b200_index_d(const b200_index* idx);
int     b200_index_nlist(const b200_index* idx);               /* 0 for flat */
/* Range sharding (SURVEY.md §8e): returned ids are id_base + local insertion position. */
int b200_index_set_id_base(b200_index* idx, int64_t id_base);
/* IVF knob the reference touches through faiss.extract_index_ivf(index).nprobe
 * (clip_back.py:357-361,368-369). */
int b200_index_set_nprobe(b200_index* idx, int nprobe);
int b200_index_get_nprobe(const b200_index* idx);
/* Batched queries (nq > 4, k <= 128) go through the wgmma scan by default; 0 forces the FMA scan
 * (kept for A/B measurements and parity tests between the paths).  Bit flags: 1 = wgmma scan on,
 * 4 = FMA scan without the bulk-copy ring, 8 = wgmma scan always in hi/lo split mode (no
 * approximate hi-only pass + exact re-score for nq > 128). */
int b200_index_set_tensor_scan(b200_index* idx, int on);
/* Queries of the last batched search whose exactness proof failed in hi-only mode and were re-run
 * in split mode (0 in the common case; diagnostic). */
int b200_index_last_hi_only_fallbacks(const b200_index* idx);
/* Plan of the last exhaustive scan launched eagerly on this handle (flat search, or the coarse step of an
 * IVF search): h_plan[4] = {kernel, queries per pass, 16-byte chunks per lane = ceil(d / 256), ring stages}.
 * kernel: 0 register FMA scan, 1 FMA scan through the bulk-copy ring, 2 wgmma split (hi/lo) scan, 3 wgmma
 * hi-only scan (queries whose proof fails are re-run in split mode).  An IVF-PQ search reports its list scan as
 * {4, sub-quantisers per CTA, CTAs per cluster, candidate warps per CTA}.  All -1 before the first scan.  A
 * replayed CUDA graph runs no host code and leaves it unchanged. */
int b200_index_last_scan_plan(const b200_index* idx, int32_t* h_plan);
/* IVF introspection used by ivf_metadata_ordering.get_old_to_new_mapping
 * (ivf_metadata_ordering.py:46-64): sizes[nlist] and, list after list, the ids in list order. */
int b200_index_ivf_lists(b200_index* idx, int64_t* h_sizes, int64_t* h_ids);
/* What a FAISS index writer needs of the quantiser.  h_info[8] = {nlist, M (0 unless IVF-PQ), by_residual,
 * has pre-transform A, has b, d (stored width), d_in (query width), nprobe}.  Each other output may be NULL:
 * h_centroids [nlist, d] fp32 (IVF-Flat: its fp16 centroids widened), h_codebook [M, 256, d / M], h_A [d, d_in],
 * h_b [d]. */
int b200_index_get_quantizer(b200_index* idx, float* h_centroids, float* h_codebook, float* h_A, float* h_b,
                             int32_t* h_info);
/* Rows [s0, s0 + n) of the store in store order (flat: insertion order; IVF: list order, after the pending rows are
 * bucketed as b200_index_finalize does), unpadded: 2 d bytes of fp16 per row, or M code bytes.  h_ids [n] (or NULL)
 * receives each slot's id (id_base + insertion id).  Either output may be NULL. */
int b200_index_copy_rows(b200_index* idx, int64_t s0, int64_t n, void* h_rows, int64_t* h_ids);

/* index.search_and_reconstruct(x, k) / index.search(x, k) with HOST buffers (the call the
 * reference makes): h_q fp32 [nq, d]; h_D fp32 [nq, k]; h_I int64 [nq, k]; h_R fp32 [nq, k, d] or
 * NULL.  Copies in, searches, copies out, synchronises. */
int b200_index_search(b200_index* idx, const float* h_q, int nq, int k,
                      float* h_D, int64_t* h_I, float* h_R);
/* Same with DEVICE buffers, asynchronous on `stream` — except that a batched search of more than 128
 * queries (hi-only tensor scan) synchronises `stream` once to read how many exactness proofs failed. */
int b200_index_search_device(b200_index* idx, const float* d_q, int nq, int k,
                             float* d_D, int64_t* d_I, float* d_R, void* stream);
/* index.range_search(x, thresh) for ONE query (reference call sites clip_filter.py:52 and clip_back.py:294): every
 * row whose inner product with h_q exceeds `thresh` — of the whole flat index, or of the `nprobe` probed lists of
 * an IVF index (FAISS IndexIVF::range_search).  At most `cap` results
 * are written (h_D/h_I, unordered); *h_count receives the true number of hits, so a caller that sees
 * *h_count > cap retries with a larger buffer. */
int b200_index_range_search(b200_index* idx, const float* h_q, float thresh, int64_t cap, float* h_D, int64_t* h_I,
                            int64_t* h_count);
/* reconstruct(id) for a batch of ids (device buffers): d_R [n, d] fp32; id -1 -> NaN row.  Flat and IVF (the IVF
 * store is in list order; an id -> slot map is built on first use). */
int b200_index_reconstruct_device(b200_index* idx, const int64_t* d_ids, int64_t n, float* d_R, void* stream);
/* d_out[i] = d_map[d_I[i]] for 0 <= d_I[i] < nmap, else -1 (device buffers, asynchronous on `stream`; d_out may be
 * d_I): an index file's own ids for the insertion ids a search returns. */
int b200_ids_map_device(const int64_t* d_I, int64_t n, const int64_t* d_map, int64_t nmap, int64_t* d_out, int device,
                        void* stream);
/* Merge G sorted candidate lists per query into one top-k (the step after the all-gather of
 * per-shard candidates, SURVEY.md §8e): d_Dg/d_Ig are [G, nq, k]; outputs [nq, k]. */
int b200_topk_merge_device(const float* d_Dg, const int64_t* d_Ig, int G, int nq, int k,
                           float* d_D, int64_t* d_I, int device, void* stream);
/* Same merge reading G packed per-shard blocks in place — block g at d_gathered + g * shard_stride_bytes holds
 * [I int64 nq*k | D fp32 nq*k] — i.e. the receive buffer of ONE all-gather whose send buffer is the block a shard's
 * b200_index_search_device wrote (d_I = block, d_D = block + nq*k*8): no pack/unpack kernels around the collective. */
int b200_topk_merge_packed_device(const void* d_gathered, int G, size_t shard_stride_bytes, int nq, int k,
                                  float* d_D, int64_t* d_I, int device, void* stream);

/* Range-sharded search across the GPUs of one box from ONE host thread (SURVEY.md §8b/§8e): shard g is a
 * b200_index on its own device holding rows [lo_g, hi_g) with id_base = lo_g; queries are replicated, every shard
 * searches on its own stream, ONE exchange of the per-shard candidates, a device merge; h_D/h_I receive the global
 * top-k.  comms == NULL: the exchange is the search epilogue itself — each shard's last kernel stores its
 * candidate block into the root device's buffer through an NVLink peer mapping (staged copies when a device pair has
 * no peer access).  comms != NULL: `nshards` ncclComm_t (comms[g] = rank g, bound to shard g's device): one
 * ncclAllGather group, the one-process-per-GPU protocol of sharded.py; NCCL is resolved with dlopen at run time.
 * The reference has no sharded search (one CPU FAISS index per process, clip_back.py:781-782); the query contract is
 * index.search (clip_back.py:362, clip_filter.py:55). */
typedef struct b200_sharded b200_sharded;
int b200_sharded_create(b200_index* const* shards, int nshards, b200_sharded** out);
int b200_sharded_destroy(b200_sharded* h);
int b200_sharded_peer_mode(const b200_sharded* h);   /* 1: candidates travel as peer stores; 0: staged copies */
int b200_sharded_search(b200_sharded* h, void* const* comms, const float* h_q, int nq, int k, float* h_D, int64_t* h_I);
/* ncclCommInitAll / ncclCommDestroy through the same run-time binding (hosts without their own NCCL bootstrap). */
int b200_nccl_comm_init_all(int n, const int* devices, void** comms_out);
int b200_nccl_comm_destroy(void* comm);

/* Duration in milliseconds (CUDA events on the launching stream) of the row-scan kernels of the
 * last search call on this handle, and how many such kernels it launched.  bench.py uses it for
 * the roofline of the dominant kernel. */
int b200_index_last_scan_ms(const b200_index* idx, float* ms, int* launches);

/* ------------------------------------------------------------------------------------------
 * Embed path.  Replaces the model object returned by all_clip.load_clip and used through
 * model.encode_image / model.encode_text in ClipMapper.__call__
 * (clip_retrieval/clip_inference/mapper.py:42-43,57-59,65-67) and KnnService.compute_query
 * (clip_back.py:230-232,244-246), fused with the L2-normalise + cast that follows each call.
 * ------------------------------------------------------------------------------------------ */
typedef struct b200_clip b200_clip;

typedef struct b200_tower_config {
  int32_t width, layers, heads, mlp;   /* transformer */
} b200_tower_config;

typedef struct b200_clip_config {
  int32_t embed_dim;         /* D: output embedding dimension */
  int32_t image_size, patch; /* 224, 14|32 */
  b200_tower_config vision;
  int32_t context_length;    /* 77 */
  int32_t vocab_size;        /* 49408 */
  b200_tower_config text;
  int32_t quick_gelu;        /* 1: x*sigmoid(1.702x) (OpenAI weights); 0: exact erf GELU (LAION) */
  int32_t max_batch;         /* activations are sized for this many samples per call */
} b200_clip_config;

typedef struct b200_tensor_view {
  const char* name;    /* open_clip / OpenAI state_dict key, e.g. "visual.transformer.resblocks.0.attn.in_proj_weight" */
  const void* data;    /* HOST pointer, contiguous */
  int32_t dtype;       /* 0 = fp32, 1 = fp16 */
  int32_t ndim;
  int64_t shape[4];
} b200_tensor_view;

#define B200_OUT_F16 1
#define B200_OUT_F32 0

/* A `text` tower config of all zeros makes an image-only handle (the image tower of a CLIP whose text tower runs
 * elsewhere, e.g. open_clip's XLM-RoBERTa models on a b200_text_encoder): no text weights or activations are
 * allocated, context_length and vocab_size are not read, load_weights needs only the visual.* tensors, and the
 * encode_text entries return B200_ERR_UNSUPPORTED. */
int b200_clip_create(const b200_clip_config* cfg, int device, b200_clip** out);
/* OpenAI's ResNet CLIPs (RN50, RN101, RN50x4, RN50x16, RN50x64; ModifiedResNet): the image tower is a stem of three
 * 3x3 convolutions and an average pool, four stages of Bottleneck blocks (layers[i] blocks, planes width * 2^i, stride
 * 1, 2, 2, 2 taken by average pools), and an attention pool of `heads` heads of 64 over the (S/32)^2 pixels plus their
 * mean.  `cfg` supplies the text tower, embed_dim, image_size (a multiple of 32), quick_gelu and max_batch; its
 * `vision` and `patch` must be zero.  load_weights reads the visual.* keys of OpenAI's state_dict (BatchNorm running
 * statistics folded into the convolutions in fp64, eps 1e-5; num_batches_tracked is ignored).  Every other
 * b200_clip_* entry works on the handle unchanged. */
typedef struct b200_resnet_config {
  int32_t layers[4];   /* Bottleneck blocks per stage */
  int32_t width;       /* stem width w: planes of stage i are w * 2^i, the attention pool has 32 w channels */
  int32_t heads;       /* attention-pool heads: 32 w / 64 */
} b200_resnet_config;
int b200_clip_create_resnet(const b200_clip_config* cfg, const b200_resnet_config* rc, int device, b200_clip** out);
/* Google's SigLIP models as open_clip builds them (ViT-B-16-SigLIP*, ViT-L-16-SigLIP-*, ViT-SO400M-14-SigLIP*): a timm
 * ViT image tower with no class token and no ln_pre, a patch embedding with a bias, and a latent-query attention pool
 * (one learned query, `vision.heads` heads, then proj, LayerNorm and an MLP of `vision.mlp` with a residual) whose
 * output is the feature; a bidirectional text tower (no causal or padding mask) pooled at position context_length - 1
 * after ln_final, with a biased Linear projection.  Every LayerNorm uses eps 1e-6, both MLPs erf GELU.  embed_dim must
 * equal vision.width and quick_gelu must be 0.  load_weights reads open_clip's keys: visual.trunk.{patch_embed.proj,
 * pos_embed, blocks.i.{norm1, attn.qkv, attn.proj, norm2, mlp.fc1, mlp.fc2}, norm, attn_pool.{latent, q, kv, proj,
 * norm, mlp.fc1, mlp.fc2}} and text.{token_embedding, positional_embedding, transformer.resblocks.i.*, ln_final,
 * text_projection}.  Every other b200_clip_* entry works on the handle unchanged. */
int b200_clip_create_siglip(const b200_clip_config* cfg, int device, b200_clip** out);
/* open_clip's ConvNeXt CLIPs (convnext_base, convnext_base_w[_320], convnext_large_d[_320], convnext_xxlarge): the image
 * tower is timm's ConvNeXt trunk (a 4x4 stride-4 patch stem + LayerNorm, four stages of depths[s] blocks at widths
 * dims[s], each stage s > 0 entered through LayerNorm + a 2x2 stride-2 convolution; a block is depthwise 7x7 conv ->
 * LayerNorm -> Linear(C, 4C) -> erf GELU -> Linear(4C, C), scaled per channel by its gamma and added to its input), then
 * the spatial mean, LayerNorm and open_clip's head: a bias-free Linear(dims[3], embed_dim) (head_mlp 0) or Linear(dims[3],
 * 2 embed_dim) + bias -> erf GELU -> bias-free Linear(2 embed_dim, embed_dim) (head_mlp 1).  Every LayerNorm of the trunk
 * uses eps.  `cfg` supplies the text tower (open_clip's standard CLIP text tower, top-level keys), embed_dim, image_size
 * (a multiple of 32), quick_gelu and max_batch; its `vision` and `patch` must be zero.  dims are multiples of 64, at most
 * 1536 for stages 0..2 and 3072 for stage 3.  load_weights reads visual.trunk.{stem.{0,1}, stages.s.downsample.{0,1}
 * (s >= 1), stages.s.blocks.j.{conv_dw, norm, mlp.fc1, mlp.fc2, gamma}, head.norm} and visual.head.proj.weight or
 * visual.head.mlp.{fc1.weight, fc1.bias, fc2.weight}; a missing one is B200_ERR_INVALID naming it.  Every other
 * b200_clip_* entry works on the handle unchanged. */
typedef struct b200_convnext_config {
  int32_t depths[4];   /* blocks per stage */
  int32_t dims[4];     /* width of each stage */
  int32_t head_mlp;    /* 0: linear projection head, 1: MLP head */
  float eps;           /* LayerNorm epsilon of the trunk (1e-6; timm's xxlarge: 1e-5) */
} b200_convnext_config;
int b200_clip_create_convnext(const b200_clip_config* cfg, const b200_convnext_config* ncfg, int device,
                              b200_clip** out);
int b200_clip_destroy(b200_clip* m);
/* Upload weights given as a state_dict in the open_clip/OpenAI key layout; converts to the
 * packed bf16 device layout.  Missing or mis-shaped tensors are an error. */
int b200_clip_load_weights(b200_clip* m, const b200_tensor_view* tensors, int n);
/* encode_image + `/= norm` + cast: d_pixels fp32 NCHW [B,3,S,S]; d_out [B,D] fp16 or fp32.
 * normalize=0 returns the raw projected features (what model.encode_image returns). */
int b200_clip_encode_image_device(b200_clip* m, const float* d_pixels, int B, void* d_out,
                                  int out_dtype, int normalize, void* stream);
/* encode_text: d_tokens int64 [B, context_length]; pooled at argmax(tokens) (EOT). */
int b200_clip_encode_text_device(b200_clip* m, const int64_t* d_tokens, int B, void* d_out,
                                 int out_dtype, int normalize, void* stream);
/* Host-buffer variants: the mapper call (H2D of the batch, forward, D2H of the embeddings). */
int b200_clip_encode_image(b200_clip* m, const float* h_pixels, int B, void* h_out, int out_dtype, int normalize);
int b200_clip_encode_text(b200_clip* m, const int64_t* h_tokens, int B, void* h_out, int out_dtype, int normalize);
/* Per-kernel-class device time (ms, CUDA events on the launching stream) accumulated over the encode
 * calls since profiling was switched on or since the previous read: gemm, attention, layernorm,
 * other; `spans` = number of timed kernel groups.  Synchronises on the events, then resets. */
int b200_clip_last_timing(b200_clip* m, float* ms_by_class /*[8]: gemm, attention, layernorm, other, then the
                             gemm share of qkv / out-proj / fc / c_proj */, int* spans);
/* Enable per-class event timing (event records between kernels; off by default); resets the sums. */
int b200_clip_set_profiling(b200_clip* m, int on);

/* Stand-alone GEMM entry used by the tests of the wgmma core:
 * C[M,N] (bf16) = act(A[M,K] (bf16, row-major) · W[N,K]^T (bf16, row-major) + bias[N] (fp32|NULL))
 *               (+ residual[M,N] bf16 | NULL).  act: 0 none, 1 quick_gelu, 2 gelu(erf). */
int b200_gemm_bf16_device(const void* d_A, const void* d_W, const float* d_bias, const void* d_residual,
                          void* d_C, int M, int N, int K, int act, int device, void* stream);

/* The same GEMM with the whole epilogue the model uses (what b200_gemm_bf16_device is a special case of), for the
 * kernel-level tests of every tile width and epilogue flavour.  Row r of the product goes to output row
 *   r                                                  (out_group == 0)
 *   (r / out_group) * (out_group + 1) + 1 + r % out_group  (out_group > 0: one cls row skipped per group)
 * and reads residual row r, or res_row_off + r % res_row_mod when res_row_mod > 0.  ld 0 means N.
 * bn: 0 = the width the library picks, else 32, 64, 128 or 256.  256 is the persistent 128 x 256 kernel of the
 * large-batch shapes.
 * flags: 0, or 2 = with bn = 256, the TMA-store epilogue whatever the grid size (the library takes it from 8 tiles
 * per SM up); it stores the same bits.  Any other bit is refused (B200_ERR_INVALID).
 * The four reserved members once carried the inputs of a LayerNorm fold that no longer exists.  They keep the
 * struct's size and layout, so callers that fill it positionally keep working, and must be NULL / 0: anything else
 * is refused (B200_ERR_INVALID) rather than ignored. */
typedef struct b200_gemm_epilogue {
  const float* bias;        /* [N] fp32 or NULL */
  const void* residual;     /* bf16, added after the activation, or NULL; may equal the output (in-place update) */
  int64_t res_ld;
  int32_t res_row_mod, res_row_off;
  int64_t out_ld;
  int32_t out_group;
  int32_t act;              /* 0 none, 1 quick_gelu, 2 gelu(erf) */
  const void* reserved0;    /* NULL */
  const void* reserved1;    /* NULL */
  int32_t reserved2;        /* 0 */
  const void* reserved3;    /* NULL */
} b200_gemm_epilogue;
int b200_gemm_bf16_ex_device(const void* d_A, const void* d_W, void* d_C, int M, int N, int K,
                             const b200_gemm_epilogue* ep, int bn, int flags, int device, void* stream);

/* Stand-alone entries of the two other embed kernels, for their parity tests:
 * LayerNorm (eps 1e-5) over rows of `w` bf16 values; multi-head attention over a fused qkv buffer
 * [B*T, 3w] (q | k | v, heads of w/heads columns) -> [B*T, w], causal != 0 adds the text mask. */
int b200_layernorm_bf16_device(const void* d_in, void* d_out, const float* d_gamma, const float* d_beta,
                               int64_t rows, int w, int device, void* stream);
int b200_attention_bf16_device(const void* d_qkv, void* d_out, int B, int T, int heads, int w, int causal,
                               int device, void* stream);
/* The ends of the two towers, for their parity tests.
 * Vision front: d_pixels fp32 NCHW [B, 3, S, S] -> d_cols bf16 [B * g * g, Kp] (g = S / p, Kp >= 3 p^2): row
 * b * g * g + py * g + px, column c * p * p + i * p + j holds pixel (c, py * p + i, px * p + j) rounded to bf16, and
 * columns >= 3 p^2 are not written.  With d_x non-NULL, row b * T of d_x bf16 [B * T, w] becomes d_cls (fp32 [w])
 * rounded to bf16 for every b (the class-token rows) and no other row is written.
 * Text front: d_x bf16 [B * T, w] row b * T + t = bf16(d_tok_emb[clamp(d_tokens[b, t], 0, vocab - 1)] + d_pos[t])
 * (d_tokens int64 [B, T], d_tok_emb bf16 [vocab, w], d_pos fp32 [T, w], w a multiple of 8); the EOT index
 * d_idx int32 [B] = the first t of the largest token of row b.
 * Tower end: d_out [B, D] = normalise(LN(x[b * T + t_b]) @ d_proj) with t_b = d_pool_idx[b] (int32), or 0 when
 * d_pool_idx is NULL; LN eps 1e-5 with fp32 d_gamma, d_beta [w]; d_proj bf16 [w, D]; d_feat fp32 [B, D] receives the
 * raw projected features; normalise is `/ |f|` with no epsilon when `normalize` (a zero row gives NaN), else none. */
int b200_vision_front_bf16_device(const float* d_pixels, int B, int S, int p, int Kp, void* d_cols, const float* d_cls,
                                  int T, int w, void* d_x, int device, void* stream);
int b200_text_embed_bf16_device(const int64_t* d_tokens, const void* d_tok_emb, const float* d_pos, void* d_x, int B,
                                int T, int w, int vocab, int device, void* stream);
int b200_token_argmax_device(const int64_t* d_tokens, int B, int T, int32_t* d_idx, int device, void* stream);
int b200_pool_ln_proj_device(const void* d_x, int B, int T, int w, const int32_t* d_pool_idx, const float* d_gamma,
                             const float* d_beta, const void* d_proj, int D, float* d_feat, void* d_out, int out_dtype,
                             int normalize, int device, void* stream);
/* The kernels of the ResNet image tower, for their parity tests.
 * Convolution: d_x NHWC bf16 [B, H, W, C] (C a multiple of 8) -> d_out [B * H * W, N] rows (ld ep->out_ld, 0 = N):
 *   ksize 3: stride 1, pad 1, as an implicit GEMM (im2col TMA loads, no im2col buffer); d_w bf16 [N, 9 * C64] with
 *            C64 = ceil(C / 64) * 64, column (3 r + s) * C64 + c = weight[n, c, r, s], zero in the padding columns;
 *            bn 0 (the library's pick), 32, 64 or 128.
 *   ksize 1: the GEMM of the rows, d_w [N, C]; bn as for b200_gemm_bf16_ex_device (256: the persistent kernel).
 *   The epilogue is b200_gemm_epilogue without row maps (out_group and res_row_mod 0); act 0 none or 3 relu, which
 *   computes relu(acc + bias + residual) with the residual added before the activation (ksize 1 also takes 1, 2).
 *   The kernel is conv3x3_bf16_wgmma_kernel.
 * Stem gather: d_pixels fp32 NCHW [B, 3, S, S] (S even) -> d_cols bf16 [B * (S/2)^2, 64], row b (S/2)^2 + oy S/2 + ox,
 *   column c * 9 + r * 3 + s = pixel (c, 2 oy - 1 + r, 2 ox - 1 + s), zero outside the image; columns 27..63 are not
 *   written.
 * Average pool: NHWC bf16 [B, H, W, C] -> [B, H / k, W / k, C] (floor), fp32 sum of each k x k window / k^2, C a
 *   multiple of 8.
 * Attention-pool tokens: d_x bf16 [B * HW, C] -> d_out bf16 [B * (HW + 1), C]: row b (HW + 1) = fp32 mean of the HW
 *   rows of sample b + d_pos[0], row b (HW + 1) + t = row b HW + t - 1 + d_pos[t] (d_pos fp32 [HW + 1, C]). */
int b200_conv_bf16_device(const void* d_x, int B, int H, int W, int C, const void* d_w, int N, int ksize, void* d_out,
                          const b200_gemm_epilogue* ep, int bn, int device, void* stream);
int b200_stem_gather_device(const float* d_pixels, int B, int S, void* d_cols, int device, void* stream);
int b200_avgpool_bf16_device(const void* d_in, int B, int H, int W, int C, int k, void* d_out, int device, void* stream);
int b200_attnpool_tokens_device(const void* d_x, int B, int HW, int C, const float* d_pos, void* d_out, int device,
                                void* stream);
/* The two kernels of SigLIP's tower ends, for their parity tests.
 * Latent-query attention pool: d_kv bf16 [B * T, 2w] (k | v, `heads` heads of hd = w / heads, hd a multiple of 8 up to
 *   128), d_q fp32 [w] -> d_out bf16 [B, w], d_out[b, h hd + j] = sum_t softmax_t(q_h . k_{b,t,h} hd^-0.5) v_{b,t,h,j},
 *   with scores, softmax and sums in fp32.
 * Text tail: d_out [B, D] = normalise(LN_eps(x[b * T + T - 1]) @ d_proj + d_bias), d_proj bf16 [w, D], d_bias fp32
 *   [D]; d_feat fp32 [B, D] receives the raw features; otherwise as b200_pool_ln_proj_device. */
int b200_latent_pool_attention_device(const void* d_kv, int B, int T, int heads, int w, const float* d_q, void* d_out,
                                      int device, void* stream);
int b200_pool_last_ln_proj_bias_device(const void* d_x, int B, int T, int w, const float* d_gamma, const float* d_beta,
                                       float eps, const void* d_proj, const float* d_bias, int D, float* d_feat,
                                       void* d_out, int out_dtype, int normalize, int device, void* stream);
/* The kernels of the ConvNeXt tower, for their parity tests.
 * Depthwise 7x7 + LayerNorm: d_x NHWC bf16 [B, H, W, C] (C a multiple of 64, at most 3072) -> d_out bf16 [B H W, C] =
 *   LN_eps(bias[c] + sum_{r,s} d_w49[7 r + s, c] x[h + r - 3, w + s - 3, c]) * gamma[c] + beta[c], zero padding, the
 *   taps summed in fp32 in the order (r, s) and the LayerNorm taken on those fp32 sums; d_w49 fp32 [49, C] (conv_dw's
 *   weight [C, 1, 7, 7] transposed); d_gamma == NULL: the convolution + bias alone (d_beta and eps unused).
 * LayerNorm + space-to-depth: d_x [B, H, W, C] (H, W even, C a multiple of 8, at most 1536) -> d_out bf16
 *   [B (H/2) (W/2), 4C], column (2 i + j) C + c = LN_eps(x[b, 2 ho + i, 2 wo + j, :])[c] gamma[c] + beta[c].
 * Head: d_x bf16 [B HW, C] -> d_pooled fp32 [B, C] = LN_eps(fp32 mean of the HW rows of sample b) gamma + beta; then
 *   with d_w1T == NULL, feat = pooled @ d_w2T fp32 [C, D]; otherwise hid = gelu_erf(pooled @ d_w1T fp32 [C, h] +
 *   d_b1[h]) into d_hid fp32 [B, h] and feat = hid @ d_w2T fp32 [h, D]; feat into d_feat fp32 [B, D], then d_out =
 *   feat / |feat| (normalize) as fp16 or fp32 (out_dtype). */
int b200_dwconv7_ln_bf16_device(const void* d_x, int B, int H, int W, int C, const float* d_w49, const float* d_bias,
                                const float* d_gamma, const float* d_beta, float eps, void* d_out, int device,
                                void* stream);
int b200_ln_s2d_bf16_device(const void* d_x, int B, int H, int W, int C, const float* d_gamma, const float* d_beta,
                            float eps, void* d_out, int device, void* stream);
int b200_convnext_head_device(const void* d_x, int B, int HW, int C, const float* d_gamma, const float* d_beta, float eps,
                              const float* d_w1T, const float* d_b1, int h, const float* d_w2T, int D, float* d_pooled,
                              float* d_hid, float* d_feat, void* d_out, int out_dtype, int normalize, int device,
                              void* stream);
/* ------------------------------------------------------------------------------------------
 * Multilingual text towers (use_mclip).  Replaces the M-CLIP text model of the query service
 * (clip_back.py:222-224,836-859: XLM-RoBERTa-Large + mean pool + LinearTransformation) and the
 * SentenceTransformer of the mapper (mapper.py:44-47,62-63: DistilBERT + mean pool + Dense), each
 * followed by normalized().  A BERT-family encoder: bidirectional attention under a key-padding mask,
 * post-LayerNorm blocks, erf GELU, masked mean pooling, a linear projection.  Head dimension 64.
 * ------------------------------------------------------------------------------------------ */
typedef struct b200_text_encoder b200_text_encoder;

typedef struct b200_text_encoder_config {
  int32_t layers, width, heads, ffn;
  int32_t vocab_size;
  int32_t max_positions;     /* rows of the position table */
  int32_t type_vocab_size;   /* rows of the token-type table; 0 = the model has none (DistilBERT) */
  int32_t position_offset;   /* position id of token t is position_offset + t (XLM-R: pad_token_id + 1 = 2) */
  float   layer_norm_eps;    /* from the model config (XLM-R-Large 1e-5, DistilBERT 1e-12) */
  int32_t out_dim;           /* projection output dimension */
  int32_t proj_bias;         /* 1: the projection has a bias */
  int32_t max_batch;         /* samples per forward (larger calls run in chunks) */
  int32_t max_tokens;        /* longest T of a call (<= 512, position_offset + max_tokens <= max_positions) */
} b200_text_encoder_config;

int b200_text_encoder_create(const b200_text_encoder_config* cfg, int device, b200_text_encoder** out);
/* The same encoder with the MLP head of open_clip's HuggingFace text towers (proj "mlp", mean pooler):
 * out = normalized(W2 · gelu_erf(W1 · mean)), W1 [hidden, width], W2 [out_dim, hidden], no biases, fp32 throughout.
 * cfg->proj_bias must be 0; load_weights then takes projection.0.weight and projection.2.weight instead of
 * projection.weight. */
int b200_text_encoder_create_mlp(const b200_text_encoder_config* cfg, int hidden, int device, b200_text_encoder** out);
int b200_text_encoder_destroy(b200_text_encoder* m);
/* Weights in the HuggingFace BERT / XLM-RoBERTa key layout without a model prefix:
 * embeddings.{word,position,token_type}_embeddings.weight, embeddings.LayerNorm.{weight,bias},
 * encoder.layer.N.attention.self.{query,key,value}.{weight,bias}, encoder.layer.N.attention.output.dense.*,
 * encoder.layer.N.attention.output.LayerNorm.*, encoder.layer.N.intermediate.dense.*, encoder.layer.N.output.dense.*,
 * encoder.layer.N.output.LayerNorm.*, and projection.weight [out_dim, width] (+ projection.bias).  Only row 0 of
 * the token-type table is used.  Missing or mis-shaped tensors are an error. */
int b200_text_encoder_load_weights(b200_text_encoder* m, const b200_tensor_view* tensors, int n);
/* d_ids int64 [B, T] right-padded, d_len int32 [B] with values 1..T (tokens of each sample; the others are never
 * attended to nor pooled).  d_out [B, out_dim] fp16 or fp32; normalize: 0 raw projected features, 1 normalized()
 * (a / |a|, a zero row stays zero).  Asynchronous on `stream`. */
int b200_text_encoder_encode_device(b200_text_encoder* m, const int64_t* d_ids, const int32_t* d_len, int B, int T,
                                    void* d_out, int out_dtype, int normalize, void* stream);
/* Host-buffer variant (lengths checked on the host); returns after the result is in h_out. */
int b200_text_encoder_encode(b200_text_encoder* m, const int64_t* h_ids, const int32_t* h_len, int B, int T,
                             void* h_out, int out_dtype, int normalize);
/* Per-kernel-class device time of the encode calls since profiling was switched on or since the previous read:
 * ms_by_class[4] = gemm, attention, layernorm, other (embedding, pooling); *launches = kernels of the last call. */
int b200_text_encoder_last_timing(b200_text_encoder* m, float* ms_by_class, int* launches);
int b200_text_encoder_set_profiling(b200_text_encoder* m, int on);

/* Stand-alone entries of the encoder kernels, for their parity tests: LayerNorm with an explicit epsilon;
 * non-causal attention where sample b sees its keys < d_len[b] (int32, 1..T) and its rows >= d_len[b] are zeros;
 * the embedding x = LN_eps((word[id] + tt0) + pos[position_offset + t]) (d_word bf16 [vocab, w], d_tt0 fp32 [w] or
 * NULL, d_pos fp32, output bf16 [B*T, w]). */
int b200_layernorm_eps_bf16_device(const void* d_in, void* d_out, const float* d_gamma, const float* d_beta,
                                   int64_t rows, int w, float eps, int device, void* stream);
int b200_attention_len_bf16_device(const void* d_qkv, const int32_t* d_len, void* d_out, int B, int T, int heads,
                                   int w, int device, void* stream);
/* d_len[b] = index of the first pad_id in row b of d_ids [B, T] (int64), T when the row has none: the token count
 * of a right-padded row, computed on the device (a row of padding only gives 0, which the encoder reads as 1).
 * Asynchronous on `stream`, on the current device. */
int b200_text_lengths_device(const int64_t* d_ids, int B, int T, int64_t pad_id, int32_t* d_len, void* stream);
/* The MLP head alone: masked mean of d_x bf16 [B*T, w] over t < d_len[b], d_hid [B, hidden] = gelu_erf(mean @ d_w1T),
 * d_feat [B, D] = d_hid @ d_w2T (d_w1T fp32 [w, hidden], d_w2T fp32 [hidden, D]: the nn.Linear weights transposed),
 * d_out [B, D] as the encoder writes it. */
int b200_mean_mlp_head_device(const void* d_x, int B, int T, int w, const int32_t* d_len, const float* d_w1T,
                              int hidden, const float* d_w2T, int D, float* d_hid, float* d_feat, void* d_out,
                              int out_dtype, int normalize, int device, void* stream);
int b200_encoder_embed_bf16_device(const int64_t* d_ids, const void* d_word, const float* d_tt0, const float* d_pos,
                                   int position_offset, const float* d_gamma, const float* d_beta, float eps,
                                   void* d_out, int B, int T, int w, int vocab, int device, void* stream);
/* The linear head alone: masked mean of d_x bf16 [B*T, w] over t < d_len[b] (clamped to 1..T), d_feat [B, D] =
 * mean @ d_projT (+ d_bias) (d_projT fp32 [w, D]: the nn.Linear weight transposed; d_bias fp32 [D] or NULL), d_out
 * [B, D] as the encoder writes it. */
int b200_mean_proj_head_device(const void* d_x, int B, int T, int w, const int32_t* d_len, const float* d_projT,
                               const float* d_bias, int D, float* d_feat, void* d_out, int out_dtype, int normalize,
                               int device, void* stream);

/* ---- image transform in front of the embed path (SURVEY §8(f) row 1) ----------------------------
 * Replaces `preprocess(PIL.Image)` as the reference calls it per image on the host
 * (clip_retrieval/clip_inference/reader.py:98-106,158-165; the object `load_clip` returns,
 * mapper.py:36-41): torchvision Resize(n_px, BICUBIC) -> CenterCrop(n_px) -> ToTensor ->
 * Normalize(mean, std), bit-exact with Pillow's 8-bit resampler and torchvision's float32 ops.
 * Input: n decoded images, RGB uint8 HWC, packed in one buffer (host or device) at byte offsets
 * h_offsets[i] with sizes h_heights[i] x h_widths[i] (host arrays).  Output: float32
 * [n, 3, n_px, n_px] on the device — the `image_tensor` layout `b200_clip_encode_image_device`
 * takes.  One batch at a time per handle; returns after the batch has been produced on `stream`. */
typedef struct b200_preproc b200_preproc;
int b200_preproc_create(int n_px, const float* mean3, const float* std3, int device, b200_preproc** out);
/* The same with the resize step chosen: B200_RESIZE_SHORTEST is the transform above (b200_preproc_create's);
 * B200_RESIZE_SQUASH is Resize((n_px, n_px), BICUBIC) with no crop — both sides scaled to n_px whatever the aspect
 * ratio (open_clip's resize_mode "squash"). */
#define B200_RESIZE_SHORTEST 0
#define B200_RESIZE_SQUASH 1
int b200_preproc_create_mode(int n_px, const float* mean3, const float* std3, int resize_mode, int device,
                             b200_preproc** out);
int b200_preproc_destroy(b200_preproc* p);
int b200_preproc_run(b200_preproc* p, const uint8_t* pixels, int pixels_on_device, const int64_t* h_offsets,
                     const int32_t* h_heights, const int32_t* h_widths, int n, float* d_out, void* stream);

/* JPEG decode on the GPU in front of the transform (SURVEY §8(f) row 1; the reference decodes with PIL in its
 * DataLoader workers, reader.py:98-106): nvJPEG (resolved with dlopen) decodes n host bitstreams into the packed
 * RGB uint8 HWC device buffer b200_preproc_run takes with pixels_on_device = 1.  b200_jpeg_info gives the sizes
 * (so the caller can lay out h_offsets) and fails on streams nvJPEG cannot parse — decode those on the host. */
typedef struct b200_jpeg b200_jpeg;
int b200_jpeg_create(int device, b200_jpeg** out);
int b200_jpeg_destroy(b200_jpeg* j);
int b200_jpeg_info(b200_jpeg* j, const uint8_t* const* h_streams, const size_t* h_sizes, int n, int32_t* h_heights,
                   int32_t* h_widths);
int b200_jpeg_decode(b200_jpeg* j, const uint8_t* const* h_streams, const size_t* h_sizes, int n, uint8_t* d_pixels,
                     const int64_t* h_offsets, const int32_t* h_heights, const int32_t* h_widths, void* stream);

/* ---- IVF training (SURVEY §8(f) row 2) --------------------------------------------------------------
 * k-means for the coarse quantiser of b200_index_create_ivfflat: the GPU counterpart of the training
 * step behind `clip-retrieval index` (clip_retrieval/clip_index.py:12-31 -> autofaiss.build_index ->
 * faiss Clustering) on the fp16 rows the writer produces (writer.py:67-87).  `niter` Lloyd iterations
 * from one seeded pick per stride of the rows; assignment = centroid of maximum inner product under
 * fp16-rounded centroids (the index's own add rule, ties to the lower id); update = mean of the
 * assigned rows (optionally L2-normalised: `spherical`); an empty cluster takes a perturbed copy of the
 * largest one (FAISS split_clusters, chosen deterministically).  d_rows: fp16 [n, d] on the device;
 * h_centroids: fp32 [nlist, d] on the host; h_sizes (optional): rows per list under the result. */
int b200_kmeans_train_f16(const void* d_rows, int64_t n, int d, int nlist, int niter, uint64_t seed, int spherical,
                          float* h_centroids, int64_t* h_sizes, int device);

/* ---- post-filters on the reconstructed rows of a search (SURVEY §8(f) row 3) ----------------------
 * b200_dedup_device replaces KnnService.get_non_uniques / connected_components_dedup
 * (clip_retrieval/clip_back.py:270-311): rows i, j are linked when their inner product exceeds
 * `threshold` (FAISS range_search semantics, strict >); d_drop[i] = 1 for every row that is not the
 * lowest-index member of its connected component (the rows the reference removes), d_labels[i]
 * (optional) = that lowest index.  d_rows: fp32 [k, d] on the device (the d_R block of
 * b200_index_search_device), k <= 4096; d_workspace: at least k * ceil(k/32) * 4 bytes.
 * b200_prompt_argmax_device replaces KnnService.get_violent_items (clip_back.py:321-324):
 * d_flag[i] = (argmax_p <row_i, prompt_p> == target), first maximum wins. */
int b200_dedup_device(const float* d_rows, int k, int d, float threshold, uint8_t* d_drop, int32_t* d_labels,
                      void* d_workspace, size_t workspace_bytes, int device, void* stream);
int b200_prompt_argmax_device(const float* d_rows, int k, int d, const float* d_prompts, int n_prompts, int target,
                              uint8_t* d_flag, int device, void* stream);

/* ---- dense fp32 MLP head on reconstructed rows (SURVEY §8(f) row 3) --------------------------------
 * Replaces the H14 NSFW detector the reference evaluates on the CPU per request:
 * clip_retrieval/h14_nsfw_model.py:15-34 (7 Linear layers 1024-1024-2048-1024-256-128-16-1, ReLU after
 * the first five, Dropout = identity in eval) as called by KnnService.get_unsafe_items
 * (clip_back.py:315-319: `safety_model.predict(embeddings)`, row unsafe iff logit > 0.5).
 * dims: [n_layers + 1] layer widths; relu: [n_layers] 0/1; weights are nn.Linear's [out, in] fp32.
 * b200_mlp_forward_device: d_x fp32 [n, dims[0]] -> d_y fp32 [n, dims[n_layers]], asynchronous on
 * `stream`; fp32 operands and accumulation (the reference's arithmetic class). */
typedef struct b200_mlp b200_mlp;
int b200_mlp_create(int n_layers, const int32_t* dims, const uint8_t* relu, int device, b200_mlp** out);
int b200_mlp_destroy(b200_mlp* m);
int b200_mlp_load_layer(b200_mlp* m, int layer, const float* h_weight, const float* h_bias);
int b200_mlp_forward_device(b200_mlp* m, const float* d_x, int n, float* d_y, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200CLIP_H */
