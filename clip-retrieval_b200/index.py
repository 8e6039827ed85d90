"""Index objects with the FAISS calling convention the reference uses.

Reference seam (SURVEY.md §8b B3): `ClipResource.image_index/text_index`
(clip_retrieval/clip_back.py:781-782) are FAISS indices created by `load_index`
(clip_back.py:589-596) and queried as
    distances, indices, embeddings = index.search_and_reconstruct(query, num_result_ids)   # :362
    D, I = index.search(x, k)                                                         # clip_filter.py:55
with `query` a C-contiguous float32 [nq, d] array.  Results are numpy arrays owned by Python:
D float32 [nq, k] descending, I int64 [nq, k] (-1 past the end), R float32 [nq, k, d].
All arithmetic happens in the CUDA library (include/b200clip.h); nothing here computes.
"""
import ctypes as C
import os
import threading
from dataclasses import dataclass

import numpy as np

from . import _lib
from ._lib import lib, check


@dataclass
class SynthSpec:
    """Seeded synthetic rows (include/b200clip.h b200_synth_spec; oracle/synth_ref.py is the CPU twin)."""

    seed: int = 1234
    clustered: bool = False
    centroid_seed: int = 7
    nlist: int = 0
    cw: int = 3
    nw: int = 1

    def c(self):
        return _lib.SynthSpecC(self.seed, 1 if self.clustered else 0, self.centroid_seed, self.nlist, self.cw, self.nw)


MAX_K = 8192   # results per query a single search supports (per-warp candidate lists live in shared memory)


def _torch():
    import torch  # device memory / streams only

    return torch


def _is_torch(x):
    return type(x).__module__.startswith("torch")


def _as_query(x, d):
    x = np.ascontiguousarray(x, dtype=np.float32)
    if x.ndim != 2:
        raise ValueError("query must be 2-D [nq, d], got shape %r" % (x.shape,))
    assert x.shape[1] == d, "query dimension %d != index dimension %d" % (x.shape[1], d)  # FAISS asserts too
    return x


def synth_rows(n, d, spec, row0=0, dtype="float16", device=0):
    """Rows row0..row0+n-1 of the synthetic set as a CUDA torch tensor (fp16 or fp32)."""
    torch = _torch()
    dt = torch.float16 if dtype in ("float16", "f16", torch.float16) else torch.float32
    out = torch.empty((n, d), dtype=dt, device="cuda:%d" % device)
    cs = spec.c()
    with torch.cuda.device(device):
        st = torch.cuda.current_stream().cuda_stream
        fn = lib.b200_synth_rows_f16 if dt == torch.float16 else lib.b200_synth_rows_f32
        check(fn(out.data_ptr(), n, d, row0, C.byref(cs), st), "synth_rows")
    return out


class _IndexBase:
    def __init__(self):
        self._h = C.c_void_p()
        self._lock = threading.Lock()

    def __del__(self):
        try:
            if self._h:
                lib.b200_index_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:  # interpreter shutdown
            pass

    # ---- FAISS attributes ----
    @property
    def ntotal(self):
        return int(lib.b200_index_ntotal(self._h))

    @property
    def d(self):
        return int(lib.b200_index_d(self._h))

    @property
    def is_trained(self):
        return True

    @property
    def id_base(self):
        return self._id_base

    @id_base.setter
    def id_base(self, v):
        check(lib.b200_index_set_id_base(self._h, int(v)), "set_id_base")
        self._id_base = int(v)

    # ---- building ----
    def reserve(self, n):
        check(lib.b200_index_reserve(self._h, int(n)), "reserve")

    def add(self, x):
        """index.add(x): x is [n, d] float16/float32 numpy (host) or a CUDA torch tensor."""
        if _is_torch(x):
            torch = _torch()
            if x.dim() != 2 or x.shape[1] != self.d:
                raise ValueError("add: expected [n, %d], got %r" % (self.d, tuple(x.shape)))
            x = x.contiguous()
            on_dev = 1 if x.is_cuda else 0
            if x.dtype == torch.float16:
                check(lib.b200_index_add_f16(self._h, x.data_ptr(), x.shape[0], on_dev), "add")
            elif x.dtype == torch.float32:
                check(lib.b200_index_add_f32(self._h, x.data_ptr(), x.shape[0], on_dev), "add")
            else:
                raise TypeError("add: dtype %s not supported (float16/float32)" % x.dtype)
            return
        x = np.asarray(x)
        if x.ndim != 2 or x.shape[1] != self.d:
            raise ValueError("add: expected [n, %d], got %r" % (self.d, x.shape))
        if x.dtype == np.float16:
            x = np.ascontiguousarray(x)
            check(lib.b200_index_add_f16(self._h, x.ctypes.data, x.shape[0], 0), "add")
        else:
            x = np.ascontiguousarray(x, dtype=np.float32)
            check(lib.b200_index_add_f32(self._h, x.ctypes.data, x.shape[0], 0), "add")

    def add_synthetic(self, n, spec, row0=0):
        cs = spec.c()
        check(lib.b200_index_add_synthetic(self._h, int(n), int(row0), C.byref(cs)), "add_synthetic")

    # ---- searching (host buffers: what the reference calls) ----
    def search(self, x, k):
        x = _as_query(x, self.d)
        if int(k) > MAX_K:
            raise ValueError("search: k=%d exceeds the supported maximum of %d results per query" % (k, MAX_K))
        nq = x.shape[0]
        D = np.empty((nq, k), dtype=np.float32)
        I = np.empty((nq, k), dtype=np.int64)
        check(lib.b200_index_search(self._h, x.ctypes.data, nq, int(k), D.ctypes.data, I.ctypes.data, None), "search")
        return D, I

    def search_and_reconstruct(self, x, k):
        x = _as_query(x, self.d)
        if int(k) > MAX_K:
            raise ValueError("search: k=%d exceeds the supported maximum of %d results per query" % (k, MAX_K))
        nq = x.shape[0]
        D = np.empty((nq, k), dtype=np.float32)
        I = np.empty((nq, k), dtype=np.int64)
        R = np.empty((nq, k, self.d), dtype=np.float32)
        check(
            lib.b200_index_search(self._h, x.ctypes.data, nq, int(k), D.ctypes.data, I.ctypes.data, R.ctypes.data),
            "search_and_reconstruct",
        )
        return D, I, R

    # ---- searching (device buffers, asynchronous on the current stream) ----
    def search_device(self, q, k, reconstruct=False, out=None):
        """q: CUDA float32 torch tensor [nq, d].  Returns (D, I[, R]) CUDA tensors.  `out=(D, I)` writes the result
        into caller-provided contiguous [nq, k] float32 / int64 tensors (e.g. views of a collective's send buffer).
        The C entry serialises concurrent calls on the handle (mutex + stream-ordered scratch reuse)."""
        torch = _torch()
        if not (q.is_cuda and q.dtype == torch.float32 and q.dim() == 2 and q.shape[1] == self.d):
            raise ValueError("search_device: q must be CUDA float32 [nq, %d]" % self.d)
        if int(k) > MAX_K:
            raise ValueError("search: k=%d exceeds the supported maximum of %d results per query" % (k, MAX_K))
        q = q.contiguous()
        nq = q.shape[0]
        if out is None:
            D = torch.empty((nq, k), dtype=torch.float32, device=q.device)
            I = torch.empty((nq, k), dtype=torch.int64, device=q.device)
        else:
            D, I = out
            if not (D.is_contiguous() and I.is_contiguous() and D.dtype == torch.float32 and I.dtype == torch.int64
                    and tuple(D.shape) == (nq, k) and tuple(I.shape) == (nq, k) and D.device == q.device and I.device == q.device):
                raise ValueError("search_device: out must be contiguous (float32 [nq,k], int64 [nq,k]) on the query's device")
        R = torch.empty((nq, k, self.d), dtype=torch.float32, device=q.device) if reconstruct else None
        st = torch.cuda.current_stream(q.device).cuda_stream
        check(
            lib.b200_index_search_device(
                self._h, q.data_ptr(), nq, int(k), D.data_ptr(), I.data_ptr(), R.data_ptr() if reconstruct else None, st
            ),
            "search_device",
        )
        return (D, I, R) if reconstruct else (D, I)

    def range_search(self, x, thresh):
        """index.range_search(x, thresh) -> (lims, D, I): every row with inner product > thresh, per
        query (clip_filter.py:52; the dedup of clip_back.py:294) — of the whole flat index, or of the `nprobe`
        probed lists of an IVF index.  Within a query results are sorted by id."""
        x = _as_query(x, self.d)
        lims = [0]
        Ds, Is = [], []
        for q in range(x.shape[0]):
            cap = 4096
            while True:
                D = np.empty(cap, dtype=np.float32)
                I = np.empty(cap, dtype=np.int64)
                cnt = C.c_int64(0)
                check(lib.b200_index_range_search(self._h, x[q].ctypes.data, float(thresh), cap, D.ctypes.data, I.ctypes.data,
                                                  C.byref(cnt)), "range_search")
                if cnt.value <= cap:
                    break
                cap = int(cnt.value)
            n = int(cnt.value)
            order = self._range_order(I[:n])
            Ds.append(D[:n][order])
            Is.append(I[:n][order])
            lims.append(lims[-1] + n)
        return (np.asarray(lims, dtype=np.uint64), np.concatenate(Ds) if Ds else np.empty(0, np.float32),
                np.concatenate(Is) if Is else np.empty(0, np.int64))

    def _range_order(self, I):
        """Order of one query's range hits: by id."""
        return np.argsort(I, kind="stable")

    def reconstruct(self, key):
        torch = _torch()
        ids = torch.tensor([int(key)], dtype=torch.int64, device="cuda:%d" % self.device)
        out = torch.empty((1, self.d), dtype=torch.float32, device=ids.device)
        st = torch.cuda.current_stream(ids.device).cuda_stream
        check(lib.b200_index_reconstruct_device(self._h, ids.data_ptr(), 1, out.data_ptr(), st), "reconstruct")
        return out[0].cpu().numpy()

    def set_tensor_scan(self, on):
        """Batched queries use the wgmma scan by default; False forces the FMA scan.  An int is passed
        through as the C ABI's bit flags (1 wgmma scan, 4 no bulk-copy ring, 8 split mode only)."""
        flags = (1 if on else 0) if isinstance(on, bool) else int(on)
        check(lib.b200_index_set_tensor_scan(self._h, flags), "set_tensor_scan")

    def last_hi_only_fallbacks(self):
        return int(lib.b200_index_last_hi_only_fallbacks(self._h))

    def last_scan_plan(self):
        """(kernel, queries per pass, chunks per lane, ring stages) of the last eager exhaustive scan; kernel 0 =
        register FMA, 1 = FMA through the bulk-copy ring, 2 = wgmma split, 3 = wgmma hi-only; an IVF-PQ search reports
        (4, sub-quantisers per CTA, CTAs per cluster, candidate warps) (include/b200clip.h)."""
        plan = np.zeros(4, dtype=np.int32)
        check(lib.b200_index_last_scan_plan(self._h, plan.ctypes.data), "last_scan_plan")
        return tuple(int(v) for v in plan)

    def last_scan_ms(self):
        ms = C.c_float(0)
        n = C.c_int(0)
        check(lib.b200_index_last_scan_ms(self._h, C.byref(ms), C.byref(n)), "last_scan_ms")
        return float(ms.value), int(n.value)


class B200FlatIndex(_IndexBase):
    """Exhaustive inner-product index over fp16 rows (FAISS IndexFlatIP / "SQfp16" semantics)."""

    def __init__(self, d, device=0):
        super().__init__()
        self._id_base = 0
        self.device = device
        check(lib.b200_index_create_flat(int(d), int(device), C.byref(self._h)), "create_flat")


class _IVFBase(_IndexBase):
    """What every inverted-file index shares: `nprobe` (the knob the reference touches through
    faiss.extract_index_ivf(index).nprobe, clip_back.py:357-361,368-369), the lists and finalize."""

    @property
    def nlist(self):
        return int(lib.b200_index_nlist(self._h))

    @property
    def nprobe(self):
        return int(lib.b200_index_get_nprobe(self._h))

    @nprobe.setter
    def nprobe(self, v):
        check(lib.b200_index_set_nprobe(self._h, int(v)), "set_nprobe")

    def finalize(self):
        check(lib.b200_index_finalize(self._h), "finalize")

    def invlists(self):
        """(sizes [nlist], ids concatenated list after list) — what
        ivf_metadata_ordering.get_old_to_new_mapping reads from FAISS invlists (:46-64)."""
        sizes = np.zeros(self.nlist, dtype=np.int64)
        ids = np.zeros(self.ntotal, dtype=np.int64)
        check(lib.b200_index_ivf_lists(self._h, sizes.ctypes.data, ids.ctypes.data), "ivf_lists")
        return sizes, ids


class B200IVFFlatIndex(_IVFBase):
    """IVF-Flat, inner product, fp16 rows (FAISS "IVF{nlist},SQfp16" / IndexIVFFlat semantics)."""

    def __init__(self, d, nlist, centroids, device=0):
        super().__init__()
        self._id_base = 0
        self.device = device
        c = np.ascontiguousarray(centroids, dtype=np.float32)
        if c.shape != (nlist, d):
            raise ValueError("centroids must be [%d, %d], got %r" % (nlist, d, c.shape))
        check(lib.b200_index_create_ivfflat(int(d), int(nlist), c.ctypes.data, int(device), C.byref(self._h)), "create_ivfflat")

    def add_with_lists(self, x, lists):
        """Append fp16 rows keeping an EXPLICIT inverted list per row (what an existing FAISS IVF file holds)."""
        x = np.ascontiguousarray(x, dtype=np.float16)
        lists = np.ascontiguousarray(lists, dtype=np.int32)
        if x.ndim != 2 or x.shape[1] != self.d or lists.shape != (x.shape[0],):
            raise ValueError("add_with_lists: expected rows [n, %d] and lists [n]" % self.d)
        check(lib.b200_index_add_assigned_f16(self._h, x.ctypes.data, x.shape[0], 0, lists.ctypes.data), "add_assigned")


class B200IVFPQIndex(_IVFBase):
    """IVF-PQ with 8-bit codes, inner product (FAISS IndexIVFPQ, optionally behind an OPQ / rotation pre-transform:
    what autofaiss writes as `OPQ{M}_{d},IVF{nlist}_HNSW32,PQ{M}x8`).  Scores are dis0 + the sum of the M table
    entries of a row's codes, in fp32 (DESIGN.md §5); the coarse step is exact where FAISS's HNSW quantiser is not.

    centroids: [nlist, d] fp32; codebook: [M, 256, d / M] fp32.  Rows are added as codes (`add_codes`); `encode`
    makes the codes and lists of float rows on the GPU: `index.add_codes(*index.encode(x))`."""

    def __init__(self, d, nlist, M, centroids, codebook, by_residual=True, device=0):
        super().__init__()
        self._id_base = 0
        self._d_code = int(d)
        self.device = device
        c = np.ascontiguousarray(centroids, dtype=np.float32)
        if c.shape != (nlist, d):
            raise ValueError("centroids must be [%d, %d], got %r" % (nlist, d, c.shape))
        if M < 1 or d % M:
            raise ValueError("M=%d must divide d=%d" % (M, d))
        cb = np.ascontiguousarray(codebook, dtype=np.float32)
        if cb.shape != (M, 256, d // M):
            raise ValueError("codebook must be [%d, 256, %d], got %r" % (M, d // M, cb.shape))
        check(lib.b200_index_create_ivfpq(int(d), int(nlist), int(M), 1 if by_residual else 0, c.ctypes.data, cb.ctypes.data,
                                          int(device), C.byref(self._h)), "create_ivfpq")

    @property
    def M(self):
        return int(lib.b200_index_pq_m(self._h))

    def add(self, x):
        raise NotImplementedError("IVF-PQ: add() takes no float rows; run the encoder first: add_codes(*index.encode(x))")

    def add_synthetic(self, n, spec, row0=0):
        raise NotImplementedError("IVF-PQ: add_synthetic() takes no float rows; run the encoder first: "
                                  "add_codes(*index.encode(x))")

    def encode(self, x, chunk=1 << 18):
        """(codes, lists) of rows x [n, d] (fp16 / fp32, numpy or a CUDA tensor; d = the query width, d_in once a
        pre-transform is set), computed on the GPU (C ABI `b200_index_encode_device`): the list of maximum inner
        product with the fp32 centroids, then per sub-quantiser the nearest codeword (squared L2) of the residual.
        codes: uint8 [n, M], numpy for numpy input, a CUDA tensor for CUDA input; lists: numpy int64 [n]."""
        torch = _torch()
        M, d = self.M, self.d
        on_dev = _is_torch(x) and x.is_cuda
        if not _is_torch(x):
            x = np.asarray(x)
            if x.dtype not in (np.float16, np.float32):
                x = x.astype(np.float32)
        if x.ndim != 2 or x.shape[1] != d:
            raise ValueError("encode: expected rows [n, %d], got %r" % (d, tuple(x.shape)))
        n = int(x.shape[0])
        dev = x.device if on_dev else torch.device("cuda", self.device)
        codes_d = torch.empty((n, M), dtype=torch.uint8, device=dev)
        lists = np.empty(n, np.int64)
        lists_d = torch.empty(min(n, chunk), dtype=torch.int32, device=dev)
        st = torch.cuda.current_stream(dev).cuda_stream
        for s in range(0, n, chunk):
            e = min(n, s + chunk)
            xc = x[s:e] if _is_torch(x) else torch.from_numpy(np.ascontiguousarray(x[s:e]))
            xc = xc.to(device=dev, dtype=torch.float32).contiguous()
            check(lib.b200_index_encode_device(self._h, xc.data_ptr(), e - s, lists_d.data_ptr(), None,
                                               codes_d[s:e].data_ptr(), st), "encode")
            lists[s:e] = lists_d[:e - s].cpu().numpy()
        return (codes_d if on_dev else codes_d.cpu().numpy()), lists

    def add_codes(self, codes, lists):
        """Append code rows [n, M] uint8 (numpy, or a CUDA uint8 torch tensor) with their inverted lists [n]."""
        lists = np.ascontiguousarray(lists, dtype=np.int32)
        M = self.M
        if _is_torch(codes):
            codes = codes.contiguous()
            if codes.dim() != 2 or codes.shape[1] != M or lists.shape != (codes.shape[0],) or str(codes.dtype) != "torch.uint8":
                raise ValueError("add_codes: expected uint8 codes [n, %d] and lists [n]" % M)
            check(lib.b200_index_add_codes(self._h, codes.data_ptr(), codes.shape[0], 1 if codes.is_cuda else 0,
                                           lists.ctypes.data), "add_codes")
            return
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        if codes.ndim != 2 or codes.shape[1] != M or lists.shape != (codes.shape[0],):
            raise ValueError("add_codes: expected codes [n, %d] and lists [n]" % M)
        check(lib.b200_index_add_codes(self._h, codes.ctypes.data, codes.shape[0], 0, lists.ctypes.data), "add_codes")

    # ---- lists in host memory (an on-disk index's memory map) ----
    @property
    def streamed(self):
        """True when the lists are served from host memory (`set_host_lists`), False when they are in HBM."""
        return getattr(self, "_host_lists", None) is not None

    def set_host_lists(self, invlists):
        """Serve the lists from host memory: `invlists` is a faiss_io.InvLists (list l: sizes[l] code rows of M bytes
        and their int64 ids, in a read-only memory map) and must describe this index's nlist lists of M-byte codes.
        Nothing is copied; the index keeps `invlists` (hence the map) alive.  Each search pass stages its probed
        lists into a device arena (C ABI `b200_index_set_host_lists`); results carry the lists' own ids and equal a
        resident load of the same lists bit for bit.  The index must hold no rows."""
        if invlists.nlist != self.nlist or invlists.d != self.M or invlists.dtype != np.uint8:
            raise ValueError("set_host_lists: %d lists of %d-byte codes for an index of nlist=%d, M=%d"
                             % (invlists.nlist, invlists.d, self.nlist, self.M))
        sizes = np.ascontiguousarray(invlists.sizes, np.int64)
        code_addr, id_addr = invlists.addresses()
        check(lib.b200_index_set_host_lists(self._h, self.nlist, sizes.ctypes.data, code_addr.ctypes.data,
                                            id_addr.ctypes.data), "set_host_lists")
        self._host_lists = invlists

    def set_stream_arena(self, nbytes):
        """Bytes per device arena of a streamed index (two arenas and as much pinned host staging); never less than
        nprobe x the largest list, which `0` selects.  Default 256 MiB."""
        check(lib.b200_index_set_stream_arena(self._h, C.c_size_t(int(nbytes))), "set_stream_arena")

    def last_stream_stats(self):
        """Streamed index, last search: {gather_ms, copy_ms, staged_bytes, passes} (host gather time, device time of
        the host-to-device copies, code bytes moved, query passes)."""
        s = np.zeros(4, np.float64)
        check(lib.b200_index_last_stream_stats(self._h, s.ctypes.data), "last_stream_stats")
        return {"gather_ms": float(s[0]), "copy_ms": float(s[1]), "staged_bytes": int(s[2]), "passes": int(s[3])}

    def _range_order(self, I):
        # a streamed index returns range hits in list-order slot, the insertion order of a resident load of its file
        return np.arange(I.size) if self.streamed else np.argsort(I, kind="stable")

    def reconstruct(self, key):
        if self.streamed:
            raise NotImplementedError("reconstruct: the lists are served from host memory and the index keeps no id -> "
                                      "list map (as FAISS's on-disk IVF without a direct map); use "
                                      "search_and_reconstruct, which decodes the rows it returns")
        return super().reconstruct(key)

    def set_pretransform(self, A, b=None):
        """Queries become A q (+ b), A [d, d_in] fp32; `d` then reports d_in (the width a caller passes)."""
        A = np.ascontiguousarray(A, dtype=np.float32)
        if A.ndim != 2 or A.shape[0] != self._d_code:
            raise ValueError("set_pretransform: A must be [%d, d_in], got %r" % (self._d_code, A.shape))
        bb = None if b is None else np.ascontiguousarray(b, dtype=np.float32).reshape(-1)
        if bb is not None and bb.shape != (A.shape[0],):
            raise ValueError("set_pretransform: b must be [%d]" % A.shape[0])
        check(lib.b200_index_set_pretransform(self._h, int(A.shape[1]), A.ctypes.data, None if bb is None else bb.ctypes.data),
              "set_pretransform")


def list_embedding_shards(path):
    """The `.npy` shards under `path` in global row order: the reference writer names them
    `img_emb_{id:0{w}d}.npy` with a fixed width per run (writer.py:22,67-87), so sorted file order is
    partition order, which is the row id order autofaiss assigns."""
    files = [path] if os.path.isfile(path) else sorted(
        os.path.join(path, f) for f in os.listdir(path) if f.endswith(".npy")
    )
    if not files:
        raise ValueError("load_index: no .npy shard under %s" % path)
    return files


def load_index(path, enable_faiss_memory_mapping=False, device=0, max_device_bytes=None):
    """Counterpart of clip_back.load_index (clip_back.py:589-596) for fp16 embedding shards.

    `path` is a `.npy` file or a folder of `.npy` shards in the layout the reference writer
    produces (`img_emb/img_emb_{i}.npy`, fp16 row-major; writer.py:67-87).  Shards are appended in
    sorted file order, which is the global row id order (SURVEY.md Appendix C).  The rows go
    straight to HBM; `enable_faiss_memory_mapping` is accepted for signature parity and ignored.
    A FAISS index file (what the reference passes: `image.index`, or a folder holding `populated.index`) is read by
    faiss_io.read_faiss_index when it is a flat / fp16 / IVF-Flat inner-product index, or an IVF-PQ one (8-bit codes,
    flat or HNSW coarse quantiser, optionally behind one OPQ / rotation pre-transform and an id map: what autofaiss
    writes for large collections) served from its codes; the file's nprobe is kept.  The lists may be in the file
    (ilar) or, for the folder `index_combiner` / FAISS merge_ondisk writes, in `merged_index.ivfdata` beside
    `populated.index` (ilod).  Other types raise NotImplementedError naming what is missing.

    Residency (IVF-PQ, either list format): the codes go to HBM when ntotal x the padded code pitch fits within
    `max_device_bytes`; otherwise the lists stay in the file's memory map and every search streams the probed ones
    (`B200IVFPQIndex.set_host_lists`).  The default budget is the free device memory at load time less the search
    scratch the index needs, so any file that fits is resident; an explicit budget lets the indices and the model of
    one ClipResource share a card, and 0 always streams.  Flat and IVF-Flat indices are always resident.  Either way
    results carry the file's ids.
    """
    del enable_faiss_memory_mapping
    from . import faiss_io

    target = path
    if os.path.isdir(path) and os.path.exists(os.path.join(path, "populated.index")):
        target = os.path.join(path, "populated.index")          # clip_back.py:591-592
    if os.path.isfile(target) and not target.endswith(".npy") and faiss_io.looks_like_faiss_index(target):
        return index_from_faiss(faiss_io.read_faiss_index(target), device=device, max_device_bytes=max_device_bytes)
    files = list_embedding_shards(path)
    first = np.load(files[0], mmap_mode="r")
    index = B200FlatIndex(first.shape[1], device=device)
    total = sum(np.load(f, mmap_mode="r").shape[0] for f in files)
    index.reserve(total)
    for f in files:
        index.add(np.load(f))
    return index


def merge_shard_results(Dg, Ig, k):
    """Merge per-shard candidates [G, nq, k] (CUDA tensors) into the global top-k [nq, k]."""
    torch = _torch()
    G, nq, kk = Dg.shape
    assert kk == k and Ig.shape == Dg.shape
    Dg = Dg.contiguous()
    Ig = Ig.contiguous()
    D = torch.empty((nq, k), dtype=torch.float32, device=Dg.device)
    I = torch.empty((nq, k), dtype=torch.int64, device=Dg.device)
    st = torch.cuda.current_stream(Dg.device).cuda_stream
    check(
        lib.b200_topk_merge_device(Dg.data_ptr(), Ig.data_ptr(), G, nq, k, D.data_ptr(), I.data_ptr(), Dg.device.index or 0, st),
        "topk_merge",
    )
    return D, I


def train_kmeans(rows, nlist, niter=10, seed=1234, spherical=False, device=0):
    """IVF coarse-quantiser training on the GPU (C ABI `b200_kmeans_train_f16`): the counterpart of the
    training step of `clip-retrieval index` (clip_index.py:12-31 -> autofaiss/faiss Clustering) over the
    fp16 rows the writer produces.  rows: np.float16/float32 [n, d] or a CUDA half tensor.
    Returns (centroids np.float32 [nlist, d], sizes np.int64 [nlist])."""
    torch = _torch()
    if _is_torch(rows):
        t = rows.detach()
    else:
        t = torch.from_numpy(np.ascontiguousarray(rows))
    dev = t.device if t.is_cuda else torch.device("cuda", device)
    t = t.to(device=dev, dtype=torch.float16).contiguous()
    n, d = t.shape
    cent = np.empty((nlist, d), np.float32)
    sizes = np.empty(nlist, np.int64)
    check(lib.b200_kmeans_train_f16(C.c_void_p(t.data_ptr()), n, d, int(nlist), int(niter), C.c_uint64(seed),
                                    1 if spherical else 0, C.c_void_p(cent.ctypes.data), C.c_void_p(sizes.ctypes.data),
                                    dev.index or 0), "kmeans_train")
    return cent, sizes


def train_pq(x, M, niter=25, seed=1234, device=0):
    """PQ codebook training on the GPU (C ABI `b200_pq_train_f32`): M independent Lloyd k-means of 256 codewords on
    the sub-vectors of x [n, d] (fp16 / fp32, numpy or CUDA tensor; n >= 256, M divides d), seeded as `train_kmeans`.
    Returns (codebook np.float32 [M, 256, d / M], sizes np.int64 [M, 256])."""
    torch = _torch()
    t = x.detach() if _is_torch(x) else torch.from_numpy(np.ascontiguousarray(x))
    dev = t.device if t.is_cuda else torch.device("cuda", device)
    t = t.to(device=dev, dtype=torch.float32).contiguous()
    n, d = t.shape
    if M < 1 or d % M:
        raise ValueError("train_pq: M=%d must divide d=%d" % (M, d))
    cb = np.empty((M, 256, d // M), np.float32)
    sizes = np.empty((M, 256), np.int64)
    check(lib.b200_pq_train_f32(C.c_void_p(t.data_ptr()), n, d, int(M), int(niter), C.c_uint64(seed),
                                C.c_void_p(cb.ctypes.data), C.c_void_p(sizes.ctypes.data), dev.index or 0), "pq_train")
    return cb, sizes


PQ_TRAIN_MAX_ROWS = 65536   # FAISS: max_points_per_centroid (256) x 256 codewords


def train_ivfpq(rows, nlist, M, niter=10, pq_niter=25, by_residual=True, seed=1234, device=0, A=None):
    """IVF-PQ training: the coarse quantiser by `train_kmeans` on the rows as fp16, then the PQ by `train_pq` on the
    residuals (the rows themselves without `by_residual`) of at most 65 536 rows picked one per stride (seeded).
    With a pre-transform A [d_out, d] both are trained on A x (FAISS IndexPreTransform::train order): the k-means rows
    are rotated chunk by chunk straight into one fp16 copy, the PQ sample in fp32.
    Separate from building so that range shards can be encoded against one replicated quantiser.
    Returns (centroids np.float32 [nlist, d], codebook np.float32 [M, 256, d / M]) in the pre-transformed width."""
    torch = _torch()
    t = rows.detach() if _is_torch(rows) else torch.from_numpy(np.ascontiguousarray(rows))
    dev = t.device if t.is_cuda else torch.device("cuda", device)
    n, d = t.shape
    if A is not None:
        d = int(np.asarray(A).shape[0])
    if M < 1 or d % M:
        raise ValueError("train_ivfpq: M=%d must divide d=%d" % (M, d))
    coarse = t if A is None else pretransform_rows(t, A, dtype="float16", device=dev.index or 0)
    cent, _ = train_kmeans(coarse, nlist, niter=niter, seed=seed, device=dev.index or 0)
    del coarse
    ns = min(n, PQ_TRAIN_MAX_ROWS)
    pick = torch.from_numpy(stride_picks(n, ns, seed)).to(t.device)
    sample = t[pick].to(device=dev, dtype=torch.float32).contiguous()
    if A is not None:
        sample = pretransform_rows(sample, A, device=dev.index or 0)
    return cent, train_pq_residuals(sample, cent, M, pq_niter=pq_niter, by_residual=by_residual, seed=seed,
                                    device=dev.index or 0)


def train_pq_residuals(sample, cent, M, pq_niter=25, by_residual=True, seed=1234, device=0):
    """The PQ step of `train_ivfpq`: `train_pq` on the residuals of `sample` (a CUDA fp32 tensor [n, d]) to their
    nearest of the centroids [nlist, d] (the rows themselves without `by_residual`).  Returns the codebook."""
    torch = _torch()
    nlist, d = np.asarray(cent).shape
    if by_residual:
        tmp = B200IVFPQIndex(d, nlist, M, cent, np.zeros((M, 256, d // M), np.float32), device=device)
        res = torch.empty_like(sample)
        st = torch.cuda.current_stream(sample.device).cuda_stream
        check(lib.b200_index_encode_device(tmp._h, sample.data_ptr(), sample.shape[0], None, res.data_ptr(), None, st),
              "encode")
        sample = res
    cb, _ = train_pq(sample, M, niter=pq_niter, seed=seed, device=device)
    return cb


OPQ_PHASES = ("rotate", "pq", "cross", "svd")


def train_opq(rows, M, d_out=None, niter=50, niter_pq=4, niter_pq_0=40, seed=1234, device=0, phases=False):
    """OPQ rotation training on the GPU (C ABI `b200_opq_train_f32`; FAISS OPQMatrix::train, DESIGN §5 (xiii)):
    A [d_out, d_in] fp32 with orthonormal rows such that the M-way PQ of A x loses less than that of x.  rows: the
    training rows [n, d_in] (fp16 / fp32, numpy or CUDA), 256 <= n <= 65 536 (pick them with `stride_picks`); d_out
    defaults to d_in and may not exceed it; M divides d_out.  Starts from the polar factor of a seeded Gaussian matrix
    (this project's rule, not FAISS's RNG); each iteration trains the PQ on x A^T (`niter_pq_0` Lloyd iterations the
    first time, `niter_pq` from the previous codebook after that) and sets A to the polar factor of decode(codes)^T X.
    Returns (A np.float32 [d_out, d_in], objective np.float32 [niter]: |x A^T - decode(codes)|^2 / n per iteration,
    before that iteration's rotation update); with phases=True also {phase: ms} over OPQ_PHASES, each phase timed
    between device synchronisations."""
    torch = _torch()
    t = rows.detach() if _is_torch(rows) else torch.from_numpy(np.ascontiguousarray(rows))
    dev = t.device if t.is_cuda else torch.device("cuda", device)
    t = t.to(device=dev, dtype=torch.float32).contiguous()
    n, d_in = t.shape
    d_out = d_in if d_out is None else int(d_out)
    if d_out > d_in:
        raise ValueError("train_opq: d_out=%d > d_in=%d (the rotation can only keep or reduce the width)" % (d_out, d_in))
    if M < 1 or d_out % M:
        raise ValueError("train_opq: M=%d must divide d_out=%d" % (M, d_out))
    A = np.empty((d_out, d_in), np.float32)
    obj = np.empty(max(0, int(niter)), np.float32)
    ph = np.zeros(4, np.float32)
    check(lib.b200_opq_train_f32(C.c_void_p(t.data_ptr()), n, d_in, d_out, int(M), int(niter), int(niter_pq),
                                 int(niter_pq_0), C.c_uint64(seed), C.c_void_p(A.ctypes.data),
                                 C.c_void_p(obj.ctypes.data) if obj.size else None,
                                 C.c_void_p(ph.ctypes.data) if phases else None, dev.index or 0), "opq_train")
    if phases:
        return A, obj, dict(zip(OPQ_PHASES, (float(v) for v in ph)))
    return A, obj


def pretransform_rows(rows, A, b=None, dtype="float32", device=0, chunk=1 << 18):
    """A x (+ b) for rows [n, d_in] (fp16 / fp32, numpy or CUDA) as a CUDA tensor [n, d_out] of `dtype` ("float32" or
    "float16"), by the encoder's pre-transform kernel (C ABI `b200_rows_pretransform_device`): the rows an index with
    this pre-transform quantises.  Rows go through `chunk` at a time, so besides the output the device holds one fp32
    chunk; numpy rows are uploaded chunk by chunk."""
    torch = _torch()
    A = np.ascontiguousarray(A, dtype=np.float32)
    d_out, d_in = A.shape
    if rows.shape[1] != d_in:
        raise ValueError("pretransform_rows: rows are %d wide, A expects %d" % (rows.shape[1], d_in))
    dev = torch.device("cuda", device)
    fp16 = dtype in ("float16", "f16", torch.float16)
    Ad = torch.from_numpy(A).to(dev)
    bd = None if b is None else torch.from_numpy(np.ascontiguousarray(b, dtype=np.float32).reshape(-1)).to(dev)
    n = int(rows.shape[0])
    out = torch.empty((n, d_out), dtype=torch.float16 if fp16 else torch.float32, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    for s in range(0, n, chunk):
        e = min(n, s + chunk)
        xc = rows[s:e] if _is_torch(rows) else torch.from_numpy(np.array(rows[s:e]))
        xc = xc.to(device=dev, dtype=torch.float32).contiguous()
        check(lib.b200_rows_pretransform_device(xc.data_ptr(), e - s, d_in, Ad.data_ptr(),
                                                None if bd is None else bd.data_ptr(), d_out, out[s:e].data_ptr(),
                                                1 if fp16 else 0, dev.index or 0, st), "pretransform")
    return out


def build_ivfpq_index(rows, nlist, M, niter=10, pq_niter=25, by_residual=True, seed=1234, nprobe=1, device=0,
                      chunk=1 << 20, opq_dim=None, opq_niter=50):
    """train + create + encode + add_codes + finalize: an IVF-PQ index over `rows` (fp16 / fp32, numpy or CUDA),
    the IVF-PQ counterpart of `build_ivf_index` (autofaiss's "IVF{nlist},PQ{M}x8").

    opq_dim (default None: no rotation) adds the OPQ step, autofaiss's "OPQ{M}_{opq_dim},IVF{nlist},PQ{M}x8": an OPQ
    rotation A [opq_dim, d] is trained (`train_opq`, M sub-quantisers) on at most 65 536 rows picked by `stride_picks`,
    then the coarse quantiser and the PQ are trained on A x (`train_ivfpq(A=...)`: FAISS IndexPreTransform::train
    order; the k-means rows take one extra fp16 copy of [n, opq_dim] on the device), A becomes the index's
    pre-transform and rows are encoded through it."""
    torch = _torch()
    dev = rows.device.index if _is_torch(rows) and rows.is_cuda else device
    A = None
    if opq_dim is not None:
        n = rows.shape[0]
        t = rows.detach() if _is_torch(rows) else torch.from_numpy(np.ascontiguousarray(rows))
        pick = torch.from_numpy(stride_picks(n, min(n, PQ_TRAIN_MAX_ROWS), seed)).to(t.device)
        A, _ = train_opq(t[pick], M, d_out=opq_dim, niter=opq_niter, seed=seed, device=dev or 0)
    cent, cb = train_ivfpq(rows, nlist, M, niter=niter, pq_niter=pq_niter, by_residual=by_residual, seed=seed,
                           device=device, A=A)
    idx = B200IVFPQIndex(cent.shape[1], nlist, M, cent, cb, by_residual=by_residual, device=dev or 0)
    if A is not None:
        idx.set_pretransform(A)
    for s in range(0, rows.shape[0], chunk):
        idx.add_codes(*idx.encode(rows[s:s + chunk]))
    idx.finalize()
    idx.nprobe = nprobe
    return idx


def stride_picks(n, count, seed):
    """One seeded row per stride: row lo_i + mix(seed ^ i * 0xD1342543DE82EF95) % (hi_i - lo_i) of the i-th of `count`
    equal strides of n rows (the initial-centroid rule of `b200_kmeans_train_f16` and `b200_pq_train_f32`)."""
    i = np.arange(count, dtype=np.uint64)
    lo = (np.arange(count, dtype=object) * n // count).astype(np.int64)
    hi = (np.arange(1, count + 1, dtype=object) * n // count).astype(np.int64)
    span = np.maximum(1, hi - lo).astype(np.uint64)
    with np.errstate(over="ignore"):
        x = np.uint64(seed) ^ (i * np.uint64(0xD1342543DE82EF95))
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        x = x ^ (x >> np.uint64(31))
    return lo + (x % span).astype(np.int64)


def build_ivf_index(rows, nlist, niter=10, seed=1234, nprobe=1, device=0):
    """train + create + add: an IVF-Flat index over `rows` (the GPU analogue of autofaiss.build_index
    for an "IVF{nlist},Flat" key, clip_index.py:24-31)."""
    cent, _ = train_kmeans(rows, nlist, niter=niter, seed=seed, device=device)
    idx = B200IVFFlatIndex(cent.shape[1], nlist, cent, device=device)
    idx.add(rows)
    idx.nprobe = nprobe
    return idx


def merge_packed_results(gathered, G, stride_bytes, nq, k):
    """Merge G packed per-shard blocks ([I int64 nq*k | D f32 nq*k], `stride_bytes` apart) read in place from
    `gathered` (a CUDA uint8 tensor: the receive buffer of the all-gather) into the global top-k [nq, k]."""
    torch = _torch()
    D = torch.empty((nq, k), dtype=torch.float32, device=gathered.device)
    I = torch.empty((nq, k), dtype=torch.int64, device=gathered.device)
    st = torch.cuda.current_stream(gathered.device).cuda_stream
    check(lib.b200_topk_merge_packed_device(gathered.data_ptr(), int(G), C.c_size_t(int(stride_bytes)), int(nq), int(k),
                                            D.data_ptr(), I.data_ptr(), gathered.device.index or 0, st), "topk_merge_packed")
    return D, I


class _IdMapped:
    """Index whose FAISS ids are not 0..n-1 (IndexIDMap, add_with_ids inside IVF lists): results are mapped on the host."""

    def __init__(self, index, id_map):
        self._index, self._map = index, np.asarray(id_map, dtype=np.int64)

    def __getattr__(self, name):
        return getattr(self._index, name)

    def _m(self, I):
        out = np.full_like(I, -1)
        ok = I >= 0
        out[ok] = self._map[I[ok]]
        return out

    def search(self, x, k):
        D, I = self._index.search(x, k)
        return D, self._m(I)

    def search_and_reconstruct(self, x, k):
        D, I, R = self._index.search_and_reconstruct(x, k)
        return D, self._m(I), R

    def range_search(self, x, thresh):
        lims, D, I = self._index.range_search(x, thresh)
        return lims, D, self._m(I)

    def search_device(self, q, k, reconstruct=False, out=None):
        """The inner index's search_device with I mapped to the file's ids on the device (C ABI b200_ids_map_device),
        in place in the returned (or the caller's `out`) I tensor."""
        torch = _torch()
        res = self._index.search_device(q, k, reconstruct=reconstruct, out=out)
        I = res[1]
        dm = getattr(self, "_dmap", None)
        if dm is None or dm.device != I.device:
            dm = self._dmap = torch.from_numpy(self._map).to(I.device)
        st = torch.cuda.current_stream(I.device).cuda_stream
        check(lib.b200_ids_map_device(I.data_ptr(), I.numel(), dm.data_ptr(), dm.numel(), I.data_ptr(),
                                      I.device.index or 0, st), "ids_map")
        return res


STREAM_SCRATCH_BYTES = 256 << 20   # search workspace a resident IVF-PQ index keeps beside its codes (default budget)


def _resident_budget(info, device):
    """Device bytes an IVF-PQ index's codes may take by default: the free memory now, less the search scratch and the
    8 bytes per row of slot ids and their inverse that a resident index keeps."""
    torch = _torch()
    free, _ = torch.cuda.mem_get_info(device)
    return free - STREAM_SCRATCH_BYTES - 8 * int(info["ntotal"])


def index_from_faiss(info, device=0, max_device_bytes=None):
    """Index from the arrays faiss_io.read_faiss_index returns (see load_index for the residency rule)."""
    d = info["d"]
    if info["kind"] == "ivfpq":
        inv = info["invlists"]
        pitch = (info["M"] + 15) // 16 * 16
        budget = _resident_budget(info, device) if max_device_bytes is None else int(max_device_bytes)
        index = B200IVFPQIndex(d, info["nlist"], info["M"], info["centroids"], info["codebook"],
                               by_residual=info["by_residual"], device=device)
        if info.get("transform") is not None:
            A, b = info["transform"]
            index.set_pretransform(A, b)
        index.nprobe = max(1, info["nprobe"])
        if inv.ntotal * pitch > budget:
            index.set_host_lists(inv)        # ids come straight from the lists
            return index if info.get("id_map") is None else _IdMapped(index, info["id_map"])
        for codes, lists in inv.chunks(1 << 22):   # rows per host-to-device chunk: the map may be a multi-GB file
            index.add_codes(codes, lists)
        index.finalize()
        ids = info["ids"]
        if not np.array_equal(ids, np.arange(len(ids), dtype=np.int64)):
            return _IdMapped(index, ids)
        return index
    ids = info["ids"]
    if info["kind"] == "flat":
        index = B200FlatIndex(d, device=device)
        index.reserve(info["ntotal"])
        rows = info["rows"]
        step = 1 << 20
        for s in range(0, rows.shape[0], step):
            index.add(np.ascontiguousarray(rows[s:s + step]))
    else:
        index = B200IVFFlatIndex(d, info["nlist"], info["centroids"], device=device)
        lists = np.repeat(np.arange(info["nlist"], dtype=np.int32), info["list_sizes"])
        index.add_with_lists(np.asarray(info["rows"], dtype=np.float16), lists)
        index.nprobe = max(1, info["nprobe"])
        index.finalize()
    if ids is not None and not np.array_equal(ids, np.arange(len(ids), dtype=np.int64)):
        return _IdMapped(index, ids)
    return index
