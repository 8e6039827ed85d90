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
/* IVF introspection used by ivf_metadata_ordering.get_old_to_new_mapping
 * (ivf_metadata_ordering.py:46-64): sizes[nlist] and, list after list, the ids in list order. */
int b200_index_ivf_lists(b200_index* idx, int64_t* h_sizes, int64_t* h_ids);

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

int b200_clip_create(const b200_clip_config* cfg, int device, b200_clip** out);
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

/* Stand-alone entries of the two other embed kernels, for their parity tests:
 * LayerNorm (eps 1e-5) over rows of `w` bf16 values; multi-head attention over a fused qkv buffer
 * [B*T, 3w] (q | k | v, heads of w/heads columns) -> [B*T, w], causal != 0 adds the text mask. */
int b200_layernorm_bf16_device(const void* d_in, void* d_out, const float* d_gamma, const float* d_beta,
                               int64_t rows, int w, int device, void* stream);
int b200_attention_bf16_device(const void* d_qkv, void* d_out, int B, int T, int heads, int w, int causal,
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
