"""`clip-retrieval index` on the GPU: the counterpart of clip_retrieval/clip_index.py, which calls autofaiss.build_index
on the `img_emb/` and `text_emb/` embedding folders and writes `image.index` / `text.index` for clip back
(clip_back.py:589-596 opens them with faiss.read_index).

Here every step runs in the CUDA library: k-means (`train_kmeans`), OPQ (`train_opq`), PQ (`train_pq`) and encoding
(`B200IVFPQIndex.encode`); the result is written by faiss_io.write_index.  The embedding shards are read through
memory maps in sorted file order, and the id of a row is its position in that order (`list_embedding_shards`).
Training samples are picked by `stride_picks` and gathered on the host: at most 256 * nlist rows for the coarse
quantiser (FAISS max_points_per_centroid) and 65 536 rows for PQ and OPQ.  For PQ keys the rows are encoded shard by shard in chunks,
so only the codes need to fit in HBM.  autofaiss's `<name>.json` infos file is not written: clip back does not read it.
"""
import math
import os
import re
import shutil
from dataclasses import dataclass

import numpy as np

from .index import (B200FlatIndex, B200IVFFlatIndex, B200IVFPQIndex, PQ_TRAIN_MAX_ROWS, list_embedding_shards,
                    pretransform_rows, stride_picks, train_kmeans, train_opq, train_pq_residuals, _torch)

KMEANS_MAX_POINTS_PER_CENTROID = 256   # FAISS ClusteringParameters::max_points_per_centroid
_UNITS = {"": 1, "K": 1 << 10, "M": 1 << 20, "G": 1 << 30, "T": 1 << 40}


def memory_bytes(v):
    """'4G' -> 4 * 2^30 (K, M, G, T are powers of 1024, an optional trailing 'B' is ignored); ints pass through."""
    if isinstance(v, (int, np.integer)):
        return int(v)
    m = re.fullmatch(r"\s*(\d+(?:\.\d+)?)\s*([KMGT]?)B?\s*", str(v).upper())
    if not m:
        raise ValueError("memory size %r: expected a number of bytes or e.g. '4G'" % (v,))
    return int(float(m.group(1)) * _UNITS[m.group(2)])


@dataclass
class IndexKey:
    """A parsed FAISS factory string of a form this engine builds."""

    key: str
    kind: str            # "flat", "ivfflat" or "ivfpq"
    nlist: int = 0
    M: int = 0           # PQ sub-quantisers (8-bit codes)
    opq_M: int = 0       # OPQ sub-quantisers; 0 = no rotation
    opq_dim: int = 0     # OPQ output width; 0 = the input width
    hnsw: int = 0        # the key's HNSW quantiser size (written as a flat quantiser)


_COMPONENT = re.compile(r"SQfp16|Flat|IVF\d+(?:_HNSW\d+)?|PQ\d+x8|OPQ\d+(?:_\d+)?")
_FORMS = ("SQfp16", "Flat", "IVF{n},Flat", "IVF{n},SQfp16", "IVF{n}[_HNSW{k}],PQ{M}x8",
          "OPQ{M'}[_{d'}],IVF{n}[_HNSW{k}],PQ{M}x8")


def parse_index_key(key):
    """Parse the factory strings this engine builds (all inner product):
        SQfp16, Flat                               flat index of fp16 rows
        IVF{n},Flat / IVF{n},SQfp16                IVF-Flat over fp16 rows
        IVF{n}[_HNSW{k}],PQ{M}x8                   IVF-PQ, 8-bit codes
        OPQ{M'}[_{d'}],IVF{n}[_HNSW{k}],PQ{M}x8    the same behind an OPQ rotation to d' columns (d' = d if absent)
    Rows are kept in fp16, the only row format this engine stores, so the `Flat` forms are built and written as their
    `SQfp16` counterparts.  An `_HNSW{k}` quantiser is probed exactly and written as a flat one.  Any other string
    raises NotImplementedError naming the component."""
    k = str(key).replace(" ", "")
    if k in ("SQfp16", "Flat"):
        return IndexKey(k, "flat")
    m = re.fullmatch(r"IVF(\d+),(?:Flat|SQfp16)", k)
    if m:
        return IndexKey(k, "ivfflat", nlist=int(m.group(1)))
    m = re.fullmatch(r"(?:OPQ(\d+)(?:_(\d+))?,)?IVF(\d+)(?:_HNSW(\d+))?,PQ(\d+)x8", k)
    if m:
        out = IndexKey(k, "ivfpq", nlist=int(m.group(3)), M=int(m.group(5)), opq_M=int(m.group(1) or 0),
                       opq_dim=int(m.group(2) or 0), hnsw=int(m.group(4) or 0))
        if out.nlist < 1 or out.M < 1 or (m.group(1) is not None and out.opq_M < 1):
            raise ValueError("index key %r: nlist, M and the OPQ M must be positive" % key)
        return out
    for comp in k.split(","):
        if not _COMPONENT.fullmatch(comp):
            raise NotImplementedError("index key %r: component %r is not built by this engine (it builds %s)"
                                      % (key, comp, ", ".join(_FORMS)))
    raise NotImplementedError("index key %r: the combination %r is not built by this engine (it builds %s)"
                              % (key, k, ", ".join(_FORMS)))


def default_index_key(n, d, max_index_memory_usage="4G"):
    """This project's rule for `index_key=None` (NOT autofaiss's selection, which is recalled and tuned by measurement):
        n < 10 000                       -> SQfp16
        nlist = 2^round(log2(4 sqrt(n)))
        n (2 d + 8) bytes fit the budget -> IVF{nlist},SQfp16
        otherwise OPQ{M}_{d},IVF{nlist}_HNSW32,PQ{M}x8 with M the largest of 256, 128, 64, 32, 16, 8 that divides d
        and for which n (M + 8) bytes fit; ValueError stating the budget needed when none does."""
    budget = memory_bytes(max_index_memory_usage)
    if n < 10000:
        return "SQfp16"
    nlist = 1 << int(math.floor(math.log2(4.0 * math.sqrt(n)) + 0.5))
    if n * (2 * d + 8) <= budget:
        return "IVF%d,SQfp16" % nlist
    ms = [M for M in (256, 128, 64, 32, 16, 8) if d % M == 0]
    for M in ms:
        if n * (M + 8) <= budget:
            return "OPQ%d_%d,IVF%d_HNSW32,PQ%dx8" % (M, d, nlist, M)
    if not ms:
        raise ValueError("no default index for d=%d: neither %d bytes of fp16 rows fit max_index_memory_usage=%d nor "
                         "does any PQ size of 8..256 divide d" % (d, n * (2 * d + 8), budget))
    raise ValueError("%d rows of d=%d need at least %d bytes (OPQ%d PQ%dx8 codes and ids) but max_index_memory_usage "
                     "is %d bytes" % (n, d, n * (ms[-1] + 8), ms[-1], ms[-1], budget))


class _Rows:
    """Rows of a numpy array, a `.npy` file or a folder of `.npy` shards (memory-mapped, sorted file order)."""

    def __init__(self, embeddings):
        if isinstance(embeddings, np.ndarray):
            self.parts = [embeddings]
        else:
            files = list(embeddings) if isinstance(embeddings, (list, tuple)) else list_embedding_shards(embeddings)
            self.parts = [np.load(f, mmap_mode="r") for f in files]
        self.parts = [p for p in self.parts if p.shape[0] > 0] or self.parts[:1]
        self.d = int(self.parts[0].shape[1])
        for p in self.parts:
            if p.ndim != 2 or p.shape[1] != self.d:
                raise ValueError("embeddings: every shard must be [n, %d], got %r" % (self.d, p.shape))
        self.off = np.concatenate([[0], np.cumsum([p.shape[0] for p in self.parts])]).astype(np.int64)
        self.n = int(self.off[-1])

    def take(self, picks):
        """Rows at the (ascending) positions `picks`, as one array."""
        picks = np.asarray(picks, np.int64)
        part = np.searchsorted(self.off, picks, side="right") - 1
        return np.concatenate([np.asarray(self.parts[i][picks[part == i] - self.off[i]]) for i in np.unique(part)])

    def chunks(self, rows):
        for p in self.parts:
            for s in range(0, p.shape[0], rows):
                yield np.array(p[s:s + rows])   # a writable copy of the mapped rows


def default_nprobe(nlist):
    """This project's rule for the nprobe stored in a written IVF file when none is given: floor(sqrt(nlist)) lists
    (64 at nlist 4096, 256 at 65 536).  autofaiss instead tunes nprobe against a speed target by measurement; clip back
    takes the file's nprobe as its baseline (clip_back.py:357-369), so pass `nprobe=` to match a tuned value."""
    return max(1, math.isqrt(int(nlist)))


def build_index(embeddings, index_key=None, max_index_memory_usage="4G", niter=10, pq_niter=25, opq_niter=50,
                by_residual=True, seed=1234, nprobe=None, chunk=1 << 18, device=0):
    """An index of this engine over `embeddings` (a folder of `.npy` shards, one `.npy` file, a list of them or a numpy
    array [n, d]) built on the GPU from a FAISS factory string (`parse_index_key`; None = `default_index_key`).
    Row i of the shards in sorted file order gets id i.  An IVF index gets `nprobe` (None = `default_nprobe(nlist)`).
    Host memory: the shards are memory-mapped and streamed `chunk` rows at a time, but the training samples are
    gathered on the host: at most 256 * nlist rows for k-means and 65 536 for PQ / OPQ, at the shards' row size
    (256 * 65 536 * 768 * 2 bytes = 24 GiB for fp16 rows at nlist 65 536).  Returns the index, ready for
    faiss_io.write_index."""
    torch = _torch()
    rows = _Rows(embeddings)
    n, d = rows.n, rows.d
    key = parse_index_key(index_key if index_key is not None else default_index_key(n, d, max_index_memory_usage))
    if key.kind == "flat":
        idx = B200FlatIndex(d, device=device)
        idx.reserve(n)
        for x in rows.chunks(chunk):
            idx.add(x)
        return idx
    if n < key.nlist:
        raise ValueError("index key %r: %d rows cannot train %d lists" % (key.key, n, key.nlist))
    nprobe = default_nprobe(key.nlist) if nprobe is None else int(nprobe)
    coarse_pick = stride_picks(n, min(n, KMEANS_MAX_POINTS_PER_CENTROID * key.nlist), seed)
    if key.kind == "ivfflat":
        cent, _ = train_kmeans(rows.take(coarse_pick), key.nlist, niter=niter, seed=seed, device=device)
        idx = B200IVFFlatIndex(d, key.nlist, cent, device=device)
        for x in rows.chunks(chunk):
            idx.add(x)
        idx.finalize()
        idx.nprobe = nprobe
        return idx
    d_code = key.opq_dim or d
    if key.opq_M and (d_code > d or d_code % key.opq_M):
        raise ValueError("index key %r: the OPQ width %d must be at most d=%d and a multiple of its M=%d"
                         % (key.key, d_code, d, key.opq_M))
    if d_code % key.M or key.M > 256:
        raise ValueError("index key %r: PQ M=%d must divide %d and be at most 256" % (key.key, key.M, d_code))
    if d_code % 8:
        raise ValueError("index key %r: the indexed width %d must be a multiple of 8 (the row width this engine's "
                         "indices take)" % (key.key, d_code))
    dev = torch.device("cuda", device)
    pq_sample = torch.from_numpy(np.ascontiguousarray(rows.take(stride_picks(n, min(n, PQ_TRAIN_MAX_ROWS), seed)),
                                                      dtype=np.float32)).to(dev)
    coarse = rows.take(coarse_pick)   # host
    A = None
    if key.opq_M:
        # FAISS IndexPreTransform::train: the rotation first, then the IVF-PQ on the rotated rows; the k-means sample
        # is rotated from the host chunk by chunk straight into fp16, the PQ sample stays fp32
        A, _ = train_opq(pq_sample, key.opq_M, d_out=d_code, niter=opq_niter, seed=seed, device=device)
        pq_sample = pretransform_rows(pq_sample, A, device=device)
        coarse = pretransform_rows(coarse, A, dtype="float16", device=device)
    cent, _ = train_kmeans(coarse, key.nlist, niter=niter, seed=seed, device=device)
    del coarse
    cb = train_pq_residuals(pq_sample, cent, key.M, pq_niter=pq_niter, by_residual=by_residual, seed=seed,
                            device=device)
    del pq_sample
    idx = B200IVFPQIndex(d_code, key.nlist, key.M, cent, cb, by_residual=by_residual, device=device)
    if A is not None:
        idx.set_pretransform(A)
    for x in rows.chunks(chunk):
        idx.add_codes(*idx.encode(x, chunk=chunk))
    idx.finalize()
    idx.nprobe = nprobe
    return idx


def clip_index(embeddings_folder, index_folder, max_index_memory_usage="4G", current_memory_available="16G",
               copy_metadata=True, image_subfolder="img_emb", text_subfolder="text_emb", nb_cores=None, index_key=None,
               nprobe=None, device=0):
    """clip_retrieval.clip_index.clip_index on the GPU, plus `index_key` (a factory string for both indices; None = this
    project's `default_index_key` per folder under max_index_memory_usage), `nprobe` (stored in the IVF files; None =
    this project's `default_nprobe(nlist)`, not autofaiss's tuned value) and `device`.  Writes
    `<index_folder>/image.index` and `text.index` (a missing embedding subfolder is skipped, as the reference's
    `quantize` does) and copies `<embeddings_folder>/metadata` to `<index_folder>/metadata`.  current_memory_available
    and nb_cores are accepted for signature parity: the host holds the training samples (see `build_index`) and one
    streaming chunk of rows, and no CPU threads do the work.  autofaiss's `<name>.json` infos file is not written (clip back does not read it)."""
    del current_memory_available, nb_cores
    from .faiss_io import write_index

    for sub, name in ((image_subfolder, "image"), (text_subfolder, "text")):
        folder = os.path.join(embeddings_folder, sub)
        if not os.path.exists(folder):
            continue
        idx = build_index(folder, index_key=index_key, max_index_memory_usage=max_index_memory_usage, nprobe=nprobe,
                          device=device)
        os.makedirs(index_folder, exist_ok=True)
        write_index(idx, os.path.join(index_folder, name + ".index"))
        del idx
    if copy_metadata:
        shutil.copytree(os.path.join(embeddings_folder, "metadata"), os.path.join(index_folder, "metadata"))
