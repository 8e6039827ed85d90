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
            order = np.argsort(I[:n], kind="stable")
            Ds.append(D[:n][order])
            Is.append(I[:n][order])
            lims.append(lims[-1] + n)
        return (np.asarray(lims, dtype=np.uint64), np.concatenate(Ds) if Ds else np.empty(0, np.float32),
                np.concatenate(Is) if Is else np.empty(0, np.int64))

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


class B200IVFFlatIndex(_IndexBase):
    """IVF-Flat, inner product, fp16 rows (FAISS "IVF{nlist},SQfp16" / IndexIVFFlat semantics).

    `nprobe` is the knob the reference touches through faiss.extract_index_ivf(index).nprobe
    (clip_back.py:357-361,368-369)."""

    def __init__(self, d, nlist, centroids, device=0):
        super().__init__()
        self._id_base = 0
        self.device = device
        c = np.ascontiguousarray(centroids, dtype=np.float32)
        if c.shape != (nlist, d):
            raise ValueError("centroids must be [%d, %d], got %r" % (nlist, d, c.shape))
        check(lib.b200_index_create_ivfflat(int(d), int(nlist), c.ctypes.data, int(device), C.byref(self._h)), "create_ivfflat")

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

    def add_with_lists(self, x, lists):
        """Append fp16 rows keeping an EXPLICIT inverted list per row (what an existing FAISS IVF file holds)."""
        x = np.ascontiguousarray(x, dtype=np.float16)
        lists = np.ascontiguousarray(lists, dtype=np.int32)
        if x.ndim != 2 or x.shape[1] != self.d or lists.shape != (x.shape[0],):
            raise ValueError("add_with_lists: expected rows [n, %d] and lists [n]" % self.d)
        check(lib.b200_index_add_assigned_f16(self._h, x.ctypes.data, x.shape[0], 0, lists.ctypes.data), "add_assigned")

    def invlists(self):
        """(sizes [nlist], ids concatenated list after list) — what
        ivf_metadata_ordering.get_old_to_new_mapping reads from FAISS invlists (:46-64)."""
        sizes = np.zeros(self.nlist, dtype=np.int64)
        ids = np.zeros(self.ntotal, dtype=np.int64)
        check(lib.b200_index_ivf_lists(self._h, sizes.ctypes.data, ids.ctypes.data), "ivf_lists")
        return sizes, ids


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


def load_index(path, enable_faiss_memory_mapping=False, device=0):
    """Counterpart of clip_back.load_index (clip_back.py:589-596) for fp16 embedding shards.

    `path` is a `.npy` file or a folder of `.npy` shards in the layout the reference writer
    produces (`img_emb/img_emb_{i}.npy`, fp16 row-major; writer.py:67-87).  Shards are appended in
    sorted file order, which is the global row id order (SURVEY.md Appendix C).  The rows go
    straight to HBM; `enable_faiss_memory_mapping` is accepted for signature parity and ignored.
    A FAISS index file (what the reference passes: `image.index`, or a folder holding `populated.index`) is read by
    faiss_io.read_faiss_index when it is a flat / fp16 / IVF-Flat inner-product index (the types that store rows);
    quantised-code indices raise NotImplementedError with the way out.
    """
    del enable_faiss_memory_mapping
    from . import faiss_io

    target = path
    if os.path.isdir(path) and os.path.exists(os.path.join(path, "populated.index")):
        target = os.path.join(path, "populated.index")          # clip_back.py:591-592
    if os.path.isfile(target) and not target.endswith(".npy") and faiss_io.looks_like_faiss_index(target):
        return index_from_faiss(faiss_io.read_faiss_index(target), device=device)
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


def index_from_faiss(info, device=0):
    """Index from the arrays faiss_io.read_faiss_index returns."""
    d, ids = info["d"], info["ids"]
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
