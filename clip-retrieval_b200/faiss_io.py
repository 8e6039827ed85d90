"""Reader and writer of FAISS index files for `load_index` and `clip_index` (clip_retrieval/clip_back.py:589-596 reads
`image.index` / `text.index` with `faiss.read_index`).

FAISS is not installable offline and /root/reference holds no index file, so this module restates the published
serialisation of faiss/impl/index_write.cpp / index_read.cpp (faiss-cpu >= 1.7.2, requirements.txt:8) from its
documented layout; it is UNVERIFIED against FAISS itself, in both directions — the tests round-trip this module's
own writers (`write_index` for a built index, the array writers below for test fixtures).  Supported (inner-product metric only — the reference builds `metric_type="ip"` indices):
    IxFI / IxF2 / IxFl   IndexFlat                      -> rows fp32
    IxSQ                 IndexScalarQuantizer, QT_fp16  -> rows fp16
    IwFl                 IndexIVFFlat (ArrayInvertedLists)
    IwSq                 IndexIVFScalarQuantizer, QT_fp16, by_residual = false
    IwPQ                 IndexIVFPQ, 8-bit codes  -> codes uint8 [n, M], served from the codes
    IHNf                 IndexHNSWFlat as the coarse quantiser of an IVF index: the graph is skipped, its storage
                         rows are the centroids (this engine probes the centroids exactly)
    IxPT                 IndexPreTransform with ONE LinearTransform (LTra: an OPQ matrix; rrot) around an IwPQ
    IxMp / IxM2          IndexIDMap / IDMap2 around one of the above
    ilar                 the inverted lists of an IVF index in the file itself (ArrayInvertedLists)
    ilod                 OnDiskInvertedLists: the lists in a separate data file (`merged_index.ivfdata` next to
                         `populated.index`, what `index_combiner` / FAISS's merge_ondisk write; DESIGN §5 (xiv))
That covers what autofaiss writes for large collections, `OPQ{M}_{d},IVF{nlist}_HNSW32,PQ{M}x8`, and the merged
on-disk form clip back serves LAION-5B from.  Still unsupported, with NotImplementedError naming the fourcc: a
top-level HNSW index, a flat IndexPQ (IxPq), 4-bit or fast-scan PQ, IVF refinement (IwQR) and longer transform
chains; re-index from the embedding shards (`load_index(<folder of .npy>)`) or rebuild as one of the above.

The lists are never copied while parsing: an IVF result holds `invlists`, an `InvLists` of per-list (size, code
address, id address) into read-only memory maps, and its "codes" / "rows" / "ids" arrays (list after list) are
built from it only when asked for.

Layout (little endian): fourcc u32; header = d i32, ntotal i64, dummy i64 x2, is_trained u8, metric_type i32
(0 = inner product, 1 = L2; metric_arg f32 follows when metric_type > 1); vectors are `size u64` + payload.
The file is parsed through a read-only memory map, so a multi-GB code file is not read into memory before the codes
are gathered into list order.

OnDiskInvertedLists record (ilod, FAISS OnDiskInvertedListsIOHook): nlist u64, code_size u64, a vector of
List {size, capacity, offset} (3 x u64), a vector of free Slot {offset, capacity} (2 x u64), the data file name as a
char vector, totsize u64.  In the data file a list's codes start at `offset` (capacity * code_size bytes) and its
int64 ids at offset + capacity * code_size.  The directory of the recorded name is always replaced by the index
file's own (FAISS's IO_FLAG_ONDISK_SAME_DIR): the name was recorded on the machine that ran the merge.
"""
import mmap
import os
import struct

import numpy as np

METRIC_INNER_PRODUCT, METRIC_L2 = 0, 1
QT_FP16 = 4   # faiss::ScalarQuantizer::QuantizerType: 8bit, 4bit, 8bit_uniform, 4bit_uniform, fp16, ...


def _fourcc(s):
    return struct.unpack("<I", s.encode("ascii"))[0]


def _fourcc_str(v):
    return struct.pack("<I", v).decode("ascii", errors="replace")


class _R:
    def __init__(self, buf, path=""):
        self.b, self.o, self.path = memoryview(buf), 0, path
        self.data = np.frombuffer(self.b, dtype=np.uint8)
        self.ntotal_at = []                      # offsets of the ntotal fields of the index headers (index_combiner)

    def take(self, fmt):
        v = struct.unpack_from("<" + fmt, self.b, self.o)
        self.o += struct.calcsize("<" + fmt)
        return v if len(v) > 1 else v[0]

    def vec(self, dtype, unit_bytes=None):
        n = self.take("Q")
        dt = np.dtype(dtype)
        nbytes = n * (unit_bytes if unit_bytes is not None else dt.itemsize)
        a = np.frombuffer(self.b, dtype=np.uint8, count=nbytes, offset=self.o)
        self.o += nbytes
        return a.view(dt)

    def raw(self, dtype, count):
        dt = np.dtype(dtype)
        a = np.frombuffer(self.b, dtype=dt, count=count, offset=self.o)
        self.o += count * dt.itemsize
        return a


def _header(r):
    d, ntotal = r.take("i"), r.take("q")
    r.take("q"); r.take("q")
    trained = r.take("B")
    metric = r.take("i")
    if metric > 1:
        r.take("f")
    return d, ntotal, bool(trained), metric


def _read_sq(r):
    qtype, _rangestat, _arg, d, code_size = r.take("i"), r.take("i"), r.take("f"), r.take("Q"), r.take("Q")
    r.vec(np.float32)   # trained
    if qtype != QT_FP16:
        raise NotImplementedError("ScalarQuantizer type %d: only QT_fp16 (4) stores the rows an fp16 engine serves" % qtype)
    if code_size != 2 * d:
        raise ValueError("QT_fp16 code size %d for d=%d" % (code_size, d))
    return d


class InvLists:
    """The inverted lists of an IVF index file, in place: list l holds sizes[l] rows of `d` entries of `dtype`, whose
    codes start at byte code_off[l] and int64 ids at id_off[l] of `data` (a read-only uint8 view of the index file's
    or the data file's memory map; the views keep the map open)."""

    def __init__(self, data, sizes, code_off, id_off, dtype, d):
        self.data, self.dtype, self.d = data, np.dtype(dtype), int(d)
        self.sizes = np.asarray(sizes, np.int64)
        self.code_off, self.id_off = np.asarray(code_off, np.int64), np.asarray(id_off, np.int64)

    @property
    def nlist(self):
        return self.sizes.size

    @property
    def ntotal(self):
        return int(self.sizes.sum())

    def addresses(self):
        """(code addresses, id addresses) as uint64 [nlist]: what b200_index_set_host_lists takes."""
        base = np.uint64(self.data.ctypes.data if self.data.size else 0)
        return base + self.code_off.astype(np.uint64), base + self.id_off.astype(np.uint64)

    def codes(self, l):
        n, w = int(self.sizes[l]), self.d * self.dtype.itemsize
        o = int(self.code_off[l])
        return self.data[o:o + n * w].view(self.dtype).reshape(n, self.d)

    def ids(self, l):
        n, o = int(self.sizes[l]), int(self.id_off[l])
        return self.data[o:o + 8 * n].view(np.int64)

    def chunks(self, rows):
        """(codes [m, d], list of each row [m]) list after list, about `rows` rows at a time (one copy per chunk)."""
        parts, lists, m = [], [], 0
        for l in np.nonzero(self.sizes)[0].tolist():
            parts.append(self.codes(l))
            lists.append(np.full(int(self.sizes[l]), l, np.int32))
            m += int(self.sizes[l])
            if m >= rows:
                yield np.concatenate(parts), np.concatenate(lists)
                parts, lists, m = [], [], 0
        if parts:
            yield np.concatenate(parts), np.concatenate(lists)

    def all_codes(self):
        nz = np.nonzero(self.sizes)[0].tolist()
        return np.concatenate([self.codes(l) for l in nz]) if nz else np.zeros((0, self.d), self.dtype)

    def all_ids(self):
        nz = np.nonzero(self.sizes)[0].tolist()
        return np.concatenate([self.ids(l) for l in nz]) if nz else np.zeros(0, np.int64)


class _Info(dict):
    """What read_faiss_index returns.  For an IVF index "rows" / "codes" (the stored rows list after list) and "ids"
    (their ids, through the id map when there is one) are concatenated from `invlists` on first access."""

    def __missing__(self, key):
        inv = dict.get(self, "invlists")
        if inv is None or key not in ("rows", "codes", "ids"):
            raise KeyError(key)
        if key == "ids":
            v = inv.all_ids()
            if dict.get(self, "id_map") is not None:
                v = self["id_map"][v]
        else:
            v = inv.all_codes()
        self[key] = v
        return v


def _map_file(path):
    """A read-only uint8 view of a whole file (empty file: an empty array)."""
    with open(path, "rb") as f:
        size = f.seek(0, 2)
        if size == 0:
            return np.zeros(0, np.uint8)
        return np.frombuffer(mmap.mmap(f.fileno(), 0, access=mmap.ACCESS_READ), dtype=np.uint8)


def _read_invlists(r, nlist_expected, code_dtype, d):
    """Inverted lists of `d` entries of `code_dtype` per row, as an InvLists into the memory map(s)."""
    tag = _fourcc_str(r.take("I"))
    if tag == "il00":
        raise ValueError("index has no inverted lists")
    if tag == "ilod":
        return _read_ondisk_invlists(r, nlist_expected, code_dtype, d)
    if tag != "ilar":
        raise NotImplementedError("inverted lists %r: only ArrayInvertedLists ('ilar') and OnDiskInvertedLists "
                                  "('ilod') are readable" % tag)
    nlist, code_size = r.take("Q"), r.take("Q")
    if nlist != nlist_expected or code_size != d * np.dtype(code_dtype).itemsize:
        raise ValueError("inverted lists: nlist %d (expected %d), code size %d for d=%d" % (nlist, nlist_expected, code_size, d))
    fmt = _fourcc_str(r.take("I"))
    sizes = np.zeros(nlist, dtype=np.int64)
    if fmt == "full":
        sizes[:] = r.vec(np.uint64).astype(np.int64)
    elif fmt == "sprs":
        pairs = r.vec(np.uint64).astype(np.int64).reshape(-1, 2)
        sizes[pairs[:, 0]] = pairs[:, 1]
    else:
        raise ValueError("inverted lists: unknown size encoding %r" % fmt)
    # ilar: each non-empty list's codes, then its ids, one list after another
    per_row = code_size + 8
    ends = r.o + np.cumsum(sizes * per_row)
    starts = ends - sizes * per_row
    if sizes.size and ends[-1] > len(r.b):
        raise ValueError("%s: the inverted lists run past the end of the file (%d bytes, %d needed)"
                         % (r.path, len(r.b), int(ends[-1])))
    r.o = int(ends[-1]) if sizes.size else r.o
    return InvLists(r.data, sizes, starts, starts + sizes * code_size, code_dtype, d)


def _read_ondisk_invlists(r, nlist_expected, code_dtype, d):
    nlist, code_size = r.take("Q"), r.take("Q")
    lists = np.array(r.vec(np.uint64, unit_bytes=24)).astype(np.int64).reshape(-1, 3)   # size, capacity, offset
    slots = r.vec(np.uint64, unit_bytes=16)
    name = bytes(r.vec(np.uint8)).decode("utf-8", errors="replace")
    totsize = r.take("Q")
    del slots                                    # free space inside the data file: nothing to serve
    width = d * np.dtype(code_dtype).itemsize
    if nlist != nlist_expected or lists.shape[0] != nlist:
        raise ValueError("%s: on-disk lists: nlist %d, %d list records (expected %d)"
                         % (r.path, nlist, lists.shape[0], nlist_expected))
    if code_size != width:
        raise ValueError("%s: on-disk lists: code size %d, the index stores %d bytes per row" % (r.path, code_size, width))
    data_path = os.path.join(os.path.dirname(os.path.abspath(r.path)), os.path.basename(name.replace("\\", "/")))
    if not os.path.isfile(data_path):
        raise ValueError("%s: the on-disk lists' data file %s (recorded as %r) is missing" % (r.path, data_path, name))
    data = _map_file(data_path)
    if data.size < totsize:
        raise ValueError("%s: data file %s is short: %d bytes, the index records %d" % (r.path, data_path, data.size, totsize))
    size, cap, off = lists[:, 0], lists[:, 1], lists[:, 2]
    bad = np.nonzero(cap < size)[0]
    if bad.size:
        l = int(bad[0])
        raise ValueError("%s: list %d has capacity %d < size %d" % (data_path, l, cap[l], size[l]))
    end = off + cap * (code_size + 8)
    bad = np.nonzero((size > 0) & ((off < 0) | (end > data.size)))[0]
    if bad.size:
        l = int(bad[0])
        raise ValueError("%s: list %d (offset %d, capacity %d) runs past the end of the file (%d bytes)"
                         % (data_path, l, off[l], cap[l], data.size))
    return InvLists(data, size, off, off + cap * code_size, code_dtype, d)


def _read_quantizer(r):
    """The coarse quantiser of an IVF index: a flat index, or an IndexHNSWFlat whose storage holds the centroids."""
    if _fourcc_str(struct.unpack_from("<I", r.b, r.o)[0]) != "IHNf":
        return _read_index(r)
    r.take("I")
    _header(r)
    r.vec(np.float64)                    # assign_probas
    r.vec(np.int32)                      # cum_nneighbor_per_level
    r.vec(np.int32)                      # levels
    r.vec(np.uint64)                     # offsets
    r.vec(np.int32)                      # neighbors
    r.take("iiiii")                      # entry_point, max_level, efConstruction, efSearch, upper_beam
    return _read_index(r)


def _read_linear_transform(r):
    """One VectorTransform of a pre-transform chain: (A [d_out, d_in] fp32, b [d_out] or None)."""
    tag = _fourcc_str(r.take("I"))
    if tag not in ("LTra", "rrot"):
        raise NotImplementedError("pre-transform %r: only a linear transform (LTra, e.g. an OPQ matrix) or a random "
                                  "rotation (rrot) is supported by load_index" % tag)
    have_bias = r.take("B")
    A = np.array(r.vec(np.float32))
    b = np.array(r.vec(np.float32))
    d_in, d_out = r.take("i"), r.take("i")
    r.take("B")                          # is_trained
    if A.size != d_in * d_out or (have_bias and b.size != d_out):
        raise ValueError("linear transform: A has %d entries, b %d, for d_in=%d d_out=%d" % (A.size, b.size, d_in, d_out))
    return A.reshape(d_out, d_in), (b if have_bias else None)


def _read_index(r):
    tag = _fourcc_str(r.take("I"))
    if tag in ("IxFI", "IxF2", "IxFl"):
        d, ntotal, _, metric = _header(r)
        xb = r.vec(np.float32)           # codes as bytes / 4 == floats: the count is in 4-byte units either way
        return {"kind": "flat", "d": d, "ntotal": ntotal, "metric": metric, "rows": np.array(xb.reshape(ntotal, d)), "ids": None}
    if tag == "IxSQ":
        d, ntotal, _, metric = _header(r)
        _read_sq(r)
        codes = r.vec(np.uint8)
        return {"kind": "flat", "d": d, "ntotal": ntotal, "metric": metric, "rows": np.array(codes.view(np.float16).reshape(ntotal, d)), "ids": None}
    if tag in ("IwFl", "IwSq"):
        r.ntotal_at.append(r.o + 4)
        d, ntotal, _, metric = _header(r)
        nlist, nprobe = r.take("Q"), r.take("Q")
        quant = _read_quantizer(r)
        if quant["kind"] != "flat":
            raise NotImplementedError("IVF coarse quantiser %r: only a flat quantiser is supported" % quant["kind"])
        dm_type = r.take("b")
        r.vec(np.int64)                  # direct map array
        if dm_type == 2:
            raise NotImplementedError("IVF direct map stored as a hash table")
        if tag == "IwSq":
            _read_sq(r)
            r.take("Q")                  # code_size
            if r.take("B"):
                raise NotImplementedError("IVF scalar quantiser with by_residual=true stores residual codes")
            dt = np.float16
        else:
            r.take("Q")                  # code_size
            dt = np.float32
        r.invlists_at = r.o
        inv = _read_invlists(r, nlist, dt, d)
        return _Info(kind="ivfflat", d=d, ntotal=ntotal, metric=metric, nlist=int(nlist), nprobe=int(nprobe),
                     centroids=np.asarray(quant["rows"], dtype=np.float32), list_sizes=inv.sizes, invlists=inv,
                     id_map=None)
    if tag == "IwPQ":
        r.ntotal_at.append(r.o + 4)
        d, ntotal, _, metric = _header(r)
        nlist, nprobe = r.take("Q"), r.take("Q")
        quant = _read_quantizer(r)
        if quant["kind"] != "flat":
            raise NotImplementedError("IVF coarse quantiser %r: only a flat or HNSW-flat quantiser is supported" % quant["kind"])
        dm_type = r.take("b")
        r.vec(np.int64)                  # direct map array
        if dm_type == 2:
            raise NotImplementedError("IVF direct map stored as a hash table")
        by_residual = bool(r.take("B"))
        code_size = r.take("Q")
        pq_d, M, nbits = r.take("Q"), r.take("Q"), r.take("Q")
        codebook = r.vec(np.float32)
        if nbits != 8:
            raise NotImplementedError("PQ with %d-bit codes: only 8-bit codes (PQ{M}x8) are served" % nbits)
        if pq_d != d or M < 1 or d % M:
            raise ValueError("PQ d=%d M=%d for an index of d=%d (M must divide d)" % (pq_d, M, d))
        if code_size != M:
            raise ValueError("IVF-PQ code size %d for M=%d (8-bit codes take M bytes)" % (code_size, M))
        if codebook.size != M * 256 * (d // M):
            raise ValueError("PQ codebook holds %d floats, expected %d" % (codebook.size, M * 256 * (d // M)))
        r.invlists_at = r.o
        inv = _read_invlists(r, nlist, np.uint8, M)
        return _Info(kind="ivfpq", d=d, ntotal=ntotal, metric=metric, nlist=int(nlist), nprobe=int(nprobe), M=int(M),
                     by_residual=by_residual, centroids=np.array(quant["rows"], dtype=np.float32),
                     codebook=np.array(codebook).reshape(M, 256, d // M), list_sizes=inv.sizes, invlists=inv,
                     id_map=None, transform=None)
    if tag == "IxPT":
        r.ntotal_at.append(r.o + 4)
        _header(r)
        nt = r.take("i")
        if nt != 1:
            raise NotImplementedError("pre-transform chain of %d transforms: load_index serves exactly one linear "
                                      "transform around an IVF-PQ index" % nt)
        A, b = _read_linear_transform(r)
        sub = _read_index(r)
        if sub["kind"] != "ivfpq":
            raise NotImplementedError("pre-transform around a %r index: load_index serves it around IVF-PQ only" % sub["kind"])
        if A.shape[0] != sub["d"]:
            raise ValueError("pre-transform outputs d=%d, the index holds d=%d" % (A.shape[0], sub["d"]))
        sub["transform"] = (A, b)
        return sub
    if tag in ("IxMp", "IxM2"):
        d, ntotal, _, metric = _header(r)
        sub = _read_index(r)
        id_map = r.vec(np.int64)
        if sub["kind"] == "flat":
            sub["ids"] = np.array(id_map)
        else:
            sub["id_map"] = np.asarray(id_map)    # the lists' ids index it ("ids" applies it)
        return sub
    raise NotImplementedError(
        "FAISS index type %r is not readable: this engine serves flat, IVF-Flat and IVF-PQ (8-bit codes, flat or HNSW "
        "coarse quantiser, at most one OPQ / rotation pre-transform, in-file or on-disk lists) files; a top-level HNSW "
        "index, a flat PQ index, 4-bit / fast-scan PQ and refinement are not served — rebuild as one of those types, or "
        "re-index from the embedding shards with load_index(<folder of .npy>) or build_ivf_index" % tag)


def _parse(path):
    with open(path, "rb") as f:
        if f.seek(0, 2) == 0:
            raise ValueError("%s is empty" % path)
        buf = mmap.mmap(f.fileno(), 0, access=mmap.ACCESS_READ)
    r = _R(buf, path)
    return r, _read_index(r)


def read_faiss_index(path):
    """Parse a FAISS index file into plain arrays (see the module docstring for the supported types).  The quantiser
    arrays are copies; an IVF index's lists stay in the file's (or its data file's) read-only memory map, which
    stays open while `invlists` or a view made from it lives."""
    _, info = _parse(path)
    if info["metric"] != METRIC_INNER_PRODUCT:
        raise NotImplementedError("FAISS index with metric %d: the search path is inner product (cosine on normalised rows)" % info["metric"])
    return info


def looks_like_faiss_index(path):
    try:
        with open(path, "rb") as f:
            head = f.read(4)
    except OSError:
        return False
    return len(head) == 4 and head[:2] in (b"Ix", b"Iw", b"IH", b"Ib", b"IB", b"IR", b"I2", b"IL")


# ---- writer: the same layout; the fixture writers (numpy arrays, for the tests) and write_index (a built index)
# share every record helper below --------------------------------------------------------------------------------
class _FileSink:
    """What the record helpers append to when writing straight to a file (the fixture writers collect a list)."""

    def __init__(self, f):
        self.f = f

    def append(self, b):
        self.f.write(b)


def _w_fourcc(out, tag):
    out.append(struct.pack("<I", _fourcc(tag)))


def _w_header(out, d, ntotal, metric):
    out.append(struct.pack("<iqqqBi", d, ntotal, 1 << 20, 1 << 20, 1, metric))


def _w_vec(out, a):
    a = np.ascontiguousarray(a)
    out.append(struct.pack("<Q", a.size))
    out.append(a.tobytes())


def _w_sq_fp16(out, d):
    """ScalarQuantizer QT_fp16 of width d (no trained parameters)."""
    out.append(struct.pack("<iifQQ", QT_FP16, 0, 0.0, d, 2 * d))
    _w_vec(out, np.zeros(0, np.float32))


def _w_flat_quantizer(out, centroids):
    """The coarse quantiser as an IndexFlatIP (IxFI) over the centroids."""
    nlist, d = centroids.shape
    _w_fourcc(out, "IxFI")
    _w_header(out, d, nlist, METRIC_INNER_PRODUCT)
    _w_vec(out, np.ascontiguousarray(centroids, dtype=np.float32).reshape(-1))


def _w_ivf_head(out, tag, d, n, nprobe, centroids, hnsw=False):
    """IndexIVF common part: header, nlist / nprobe, coarse quantiser, an empty direct map."""
    _w_fourcc(out, tag)
    _w_header(out, d, n, METRIC_INNER_PRODUCT)
    out.append(struct.pack("<QQ", centroids.shape[0], nprobe))
    if hnsw:
        _w_hnsw_flat(out, centroids)
    else:
        _w_flat_quantizer(out, centroids)
    out.append(struct.pack("<b", 0))
    _w_vec(out, np.zeros(0, np.int64))


def _w_pretransform(out, A, b, n, tag="LTra"):
    """IndexPreTransform head with one LinearTransform (A [d_out, d_in], b [d_out] or None); the sub-index follows."""
    A = np.ascontiguousarray(A, dtype=np.float32)
    _w_fourcc(out, "IxPT")
    _w_header(out, A.shape[1], n, METRIC_INNER_PRODUCT)
    out.append(struct.pack("<i", 1))
    out.append(struct.pack("<IB", _fourcc(tag), 0 if b is None else 1))
    _w_vec(out, A.reshape(-1))
    _w_vec(out, np.zeros(0, np.float32) if b is None else np.asarray(b, np.float32))
    out.append(struct.pack("<iiB", A.shape[1], A.shape[0], 1))


def _w_invlists_head(out, nlist, code_size, sizes, sparse_sizes=False):
    """ArrayInvertedLists up to the list contents (then per non-empty list: its codes, then its int64 ids)."""
    sizes = np.asarray(sizes).astype(np.uint64)
    out.append(struct.pack("<I", _fourcc("ilar")))
    out.append(struct.pack("<QQ", nlist, code_size))
    if sparse_sizes:
        out.append(struct.pack("<I", _fourcc("sprs")))
        nz = np.nonzero(sizes)[0]
        _w_vec(out, np.stack([nz.astype(np.uint64), sizes[nz]], axis=1).reshape(-1))
    else:
        out.append(struct.pack("<I", _fourcc("full")))
        _w_vec(out, sizes)


def _w_invlists(out, nlist, code_size, codes, ids, assign, sparse_sizes):
    assign = np.asarray(assign, dtype=np.int64)
    sizes = np.bincount(assign, minlength=nlist).astype(np.uint64)
    _w_invlists_head(out, nlist, code_size, sizes, sparse_sizes)
    order = np.argsort(assign, kind="stable")
    off = 0
    for l in range(nlist):
        m = int(sizes[l])
        if m:
            sel = order[off:off + m]
            out.append(codes[sel].tobytes())
            out.append(ids[sel].tobytes())
            off += m


def write_flat(path, rows, metric=METRIC_INNER_PRODUCT, fp16=False, id_map=None):
    rows = np.ascontiguousarray(rows, dtype=np.float16 if fp16 else np.float32)
    n, d = rows.shape
    out = []
    if id_map is not None:
        _w_fourcc(out, "IxMp")
        _w_header(out, d, n, metric)
    if fp16:
        _w_fourcc(out, "IxSQ")
        _w_header(out, d, n, metric)
        _w_sq_fp16(out, d)
        _w_vec(out, rows.view(np.uint8).reshape(-1))
    else:
        _w_fourcc(out, {0: "IxFI", 1: "IxF2"}.get(metric, "IxFl"))
        _w_header(out, d, n, metric)
        _w_vec(out, rows.reshape(-1))
    if id_map is not None:
        _w_vec(out, np.asarray(id_map, dtype=np.int64))
    with open(path, "wb") as f:
        f.write(b"".join(out))


def write_ivfflat(path, centroids, rows, assign, ids=None, nprobe=1, fp16=False, sparse_sizes=False):
    centroids = np.ascontiguousarray(centroids, dtype=np.float32)
    rows = np.ascontiguousarray(rows, dtype=np.float16 if fp16 else np.float32)
    nlist, d = centroids.shape
    n = rows.shape[0]
    ids = np.arange(n, dtype=np.int64) if ids is None else np.asarray(ids, dtype=np.int64)
    out = []
    _w_ivf_head(out, "IwSq" if fp16 else "IwFl", d, n, nprobe, centroids)
    if fp16:
        _w_sq_fp16(out, d)
        out.append(struct.pack("<QB", 2 * d, 0))
    else:
        out.append(struct.pack("<Q", 4 * d))
    _w_invlists(out, nlist, rows.dtype.itemsize * d, rows, ids, assign, sparse_sizes)
    with open(path, "wb") as f:
        f.write(b"".join(out))


def _w_hnsw_flat(out, centroids):
    """An IndexHNSWFlat over the centroids: a one-level graph whose neighbour slots are empty (-1); readers skip it."""
    nlist, d = centroids.shape
    out.append(struct.pack("<I", _fourcc("IHNf")))
    _w_header(out, d, nlist, METRIC_INNER_PRODUCT)
    _w_vec(out, np.array([1.0], np.float64))                        # assign_probas
    _w_vec(out, np.array([0, 64], np.int32))                        # cum_nneighbor_per_level (2 * HNSW32 at level 0)
    _w_vec(out, np.ones(nlist, np.int32))                           # levels
    _w_vec(out, (np.arange(nlist + 1) * 64).astype(np.uint64))      # offsets
    _w_vec(out, np.full(nlist * 64, -1, np.int32))                  # neighbors
    out.append(struct.pack("<iiiii", 0, 0, 40, 16, 1))              # entry_point, max_level, efConstruction, efSearch, upper_beam
    _w_flat_quantizer(out, centroids)


def _w_ivfpq_params(out, d, M, by_residual, codebook, nbits=8, code_size=None, pq_d=None):
    """What IwPQ adds after the IVF head: by_residual, code size, the ProductQuantizer."""
    out.append(struct.pack("<BQ", 1 if by_residual else 0, M if code_size is None else code_size))
    out.append(struct.pack("<QQQ", d if pq_d is None else pq_d, M, nbits))
    _w_vec(out, np.ascontiguousarray(codebook, dtype=np.float32).reshape(-1))


def write_ivfpq(path, centroids, codebook, codes, assign, ids=None, nprobe=1, by_residual=True, transform=None,
                transform_tag="LTra", hnsw=False, sparse_sizes=False, id_map=None, nbits=8, code_size=None, pq_d=None):
    """IndexIVFPQ in the layout read above (test fixtures).  codebook [M, 256, d / M]; codes [n, M] uint8 with list
    `assign[i]`; transform = (A [d, d_in], b or None) wraps it in IxPT (`transform_tag` LTra or rrot); hnsw = an IHNf
    quantiser; id_map wraps everything in IxMp.  nbits / code_size / pq_d override the header fields (refusal tests)."""
    codes = np.ascontiguousarray(codes, dtype=np.uint8)
    n, M = codes.shape
    ids = np.arange(n, dtype=np.int64) if ids is None else np.asarray(ids, dtype=np.int64)
    out = []
    if id_map is not None:
        _w_fourcc(out, "IxMp")
        _w_header(out, transform[0].shape[1] if transform is not None else centroids.shape[1], n, METRIC_INNER_PRODUCT)
    nlist = _w_ivfpq_head(out, centroids, codebook, n, M, nprobe, by_residual, transform, transform_tag, hnsw, nbits,
                          code_size, pq_d)
    _w_invlists(out, nlist, M if code_size is None else code_size, codes, ids, assign, sparse_sizes)
    if id_map is not None:
        _w_vec(out, np.asarray(id_map, dtype=np.int64))
    with open(path, "wb") as f:
        f.write(b"".join(out))


def _w_ivfpq_head(out, centroids, codebook, n, M, nprobe, by_residual, transform, transform_tag="LTra", hnsw=False,
                  nbits=8, code_size=None, pq_d=None):
    """An IVF-PQ index up to its inverted lists (inside IxPT when `transform` is set).  Returns nlist."""
    centroids = np.ascontiguousarray(centroids, dtype=np.float32)
    nlist, d = centroids.shape
    if transform is not None:
        _w_pretransform(out, transform[0], transform[1], n, transform_tag)
    _w_ivf_head(out, "IwPQ", d, n, nprobe, centroids, hnsw=hnsw)
    _w_ivfpq_params(out, d, M, by_residual, np.ascontiguousarray(codebook, dtype=np.float32), nbits, code_size, pq_d)
    return nlist


def _w_ondisk_record(out, nlist, code_size, lists, slots, filename, totsize):
    """OnDiskInvertedLists (ilod): lists [nlist, 3] (size, capacity, offset), slots [s, 2] (offset, capacity)."""
    out.append(struct.pack("<I", _fourcc("ilod")))
    out.append(struct.pack("<QQ", nlist, code_size))
    lists = np.ascontiguousarray(lists, dtype=np.uint64).reshape(-1, 3)
    out.append(struct.pack("<Q", lists.shape[0]))
    out.append(lists.tobytes())
    slots = np.ascontiguousarray(slots, dtype=np.uint64).reshape(-1, 2)
    out.append(struct.pack("<Q", slots.shape[0]))
    out.append(slots.tobytes())
    name = filename.encode("utf-8")
    out.append(struct.pack("<Q", len(name)))
    out.append(name)
    out.append(struct.pack("<Q", totsize))


def write_ivfpq_ondisk(folder, centroids, codebook, codes, assign, ids=None, nprobe=1, by_residual=True, transform=None,
                       hnsw=False, spare=None, recorded_dir=None, code_size=None, data_bytes=None, lists_override=None):
    """An on-disk IndexIVFPQ as FAISS's merge_ondisk leaves it (test fixtures): `folder`/populated.index with an ilod
    record and `folder`/merged_index.ivfdata holding, list after list, each list's codes then its ids.  spare[l]
    (default 0) rows of unused capacity follow list l's rows (capacity = size + spare: the id address then lies
    past the spare codes), and one free slot is recorded after the last list.  The record names the data file in
    `recorded_dir` (default: `folder`), as a merge run elsewhere does.  code_size / data_bytes / lists_override
    overwrite the record's code size, truncate the data file, or replace the (size, capacity, offset) triples
    (refusal tests).  Returns the (size, capacity, offset) triples written."""
    codes = np.ascontiguousarray(codes, dtype=np.uint8)
    n, M = codes.shape
    nlist = np.asarray(centroids).shape[0]
    ids = np.arange(n, dtype=np.int64) if ids is None else np.asarray(ids, dtype=np.int64)
    assign = np.asarray(assign, dtype=np.int64)
    spare = np.zeros(nlist, np.int64) if spare is None else np.asarray(spare, np.int64)
    order = np.argsort(assign, kind="stable")
    sizes = np.bincount(assign, minlength=nlist).astype(np.int64)
    os.makedirs(folder, exist_ok=True)
    data_path = os.path.join(folder, "merged_index.ivfdata")
    triples = np.zeros((nlist, 3), np.int64)
    with open(data_path, "wb") as f:
        off, pos = 0, 0
        for l in range(nlist):
            m, cap = int(sizes[l]), int(sizes[l] + spare[l])
            sel = order[pos:pos + m]
            pos += m
            triples[l] = (m, cap, off)
            f.write(codes[sel].tobytes() + bytes((cap - m) * M))
            f.write(ids[sel].tobytes() + bytes((cap - m) * 8))
            off += cap * (M + 8)
        totsize = off
        f.write(bytes(64))                       # one free slot past the last list
    if data_bytes is not None:
        os.truncate(data_path, data_bytes)
    if lists_override is not None:
        triples = np.asarray(lists_override, np.int64)
    out = []
    _w_ivfpq_head(out, centroids, codebook, n, M, nprobe, by_residual, transform, hnsw=hnsw)
    name = os.path.join(recorded_dir if recorded_dir is not None else os.path.abspath(folder), "merged_index.ivfdata")
    _w_ondisk_record(out, nlist, M if code_size is None else code_size, triples, np.array([[totsize, 64]]), name,
                     totsize + 64)
    with open(os.path.join(folder, "populated.index"), "wb") as f:
        f.write(b"".join(out))
    return triples


def index_combiner(input_folder, output_folder):
    """clip_retrieval.clip_back_prepro.index_combiner on the host: merge the IVF index parts under `input_folder`
    (the files whose name contains "index", in sorted order) into `output_folder`/merged_index.ivfdata and
    `output_folder`/populated.index, what FAISS's merge_ondisk(shift_ids=False) writes and `load_index(output_folder)`
    serves.  The data file holds one list after another, each the parts' rows of that list in file order (codes,
    then ids), capacity = size, ids kept as stored; populated.index is the first part's header with ntotal = the sum
    and an ilod record.  Works list by list from the parts' memory maps, so host memory stays bounded by one list.
    Refuses parts whose nlist, d, M, by_residual, centroids, codebook or pre-transform differ from the first part's
    (merging them would silently mix incompatible codes), and parts inside an id map (IxMp: the merge moves list ids,
    not the map)."""
    names = sorted(f for f in os.listdir(input_folder) if "index" in f)
    files = [os.path.join(input_folder, f) for f in names if os.path.isfile(os.path.join(input_folder, f))]
    if not files:
        raise ValueError("index_combiner: no file whose name contains 'index' under %s" % input_folder)
    parts = []
    for p in files:
        r, info = _parse(p)
        if info["kind"] == "flat":
            raise ValueError("index_combiner: %s is a flat index; only IVF indices have lists to merge" % p)
        if info.get("id_map") is not None:
            raise ValueError("index_combiner: %s is wrapped in an id map (IxMp); merging lists would detach the ids "
                             "from the map" % p)
        parts.append((p, r, info))
    p0, r0, i0 = parts[0]

    def fields(info):
        t = info.get("transform")
        return {"kind": info["kind"], "nlist": info["nlist"], "d": info["d"], "M": info.get("M"),
                "by_residual": info.get("by_residual"), "centroids": info["centroids"].tobytes(),
                "codebook": None if info.get("codebook") is None else info["codebook"].tobytes(),
                "pre-transform": None if t is None else (t[0].tobytes(), None if t[1] is None else t[1].tobytes())}

    f0 = fields(i0)
    for p, _, info in parts[1:]:
        f = fields(info)
        for key in f0:
            if f[key] != f0[key]:
                raise ValueError("index_combiner: %s differs from %s in its %s; parts must share one trained quantiser"
                                 % (p, p0, key))
    nlist, inv0 = i0["nlist"], i0["invlists"]
    width = inv0.d * inv0.dtype.itemsize
    os.makedirs(output_folder, exist_ok=True)
    data_path = os.path.abspath(os.path.join(output_folder, "merged_index.ivfdata"))
    triples = np.zeros((nlist, 3), np.int64)
    off = 0
    with open(data_path, "wb") as f:
        for l in range(nlist):
            invs = [info["invlists"] for _, _, info in parts]
            m = sum(int(inv.sizes[l]) for inv in invs)
            triples[l] = (m, m, off)
            if m:
                for inv in invs:
                    if inv.sizes[l]:
                        f.write(inv.codes(l).data)
                for inv in invs:
                    if inv.sizes[l]:
                        f.write(inv.ids(l).data)
            off += m * (width + 8)
    total = int(triples[:, 0].sum())
    head = bytearray(r0.b[:r0.invlists_at])
    for at in r0.ntotal_at:
        struct.pack_into("<q", head, at, total)
    out = [bytes(head)]
    _w_ondisk_record(out, nlist, width, triples, np.zeros((0, 2)), data_path, off)
    with open(os.path.join(output_folder, "populated.index"), "wb") as f:
        f.write(b"".join(out))
    return os.path.join(output_folder, "populated.index")


class _StoreReader:
    """Sequential reads of an index's row store (or of its slot ids) through a window of `chunk` slots."""

    def __init__(self, index, chunk, width, ids):
        self.index, self.chunk, self.width, self.ids = index, max(1, int(chunk)), width, ids
        self.w0 = self.w1 = 0
        self.buf = None

    def write(self, out, a, b):
        from ._lib import lib, check

        while a < b:
            if not (self.w0 <= a < self.w1):
                self.w0, self.w1 = a, min(self.index.ntotal, a + self.chunk)
                m = self.w1 - self.w0
                if self.ids:
                    self.buf = np.empty(m, np.int64)
                    check(lib.b200_index_copy_rows(self.index._h, self.w0, m, None, self.buf.ctypes.data), "copy_rows")
                else:
                    self.buf = np.empty((m, self.width), np.uint8)
                    check(lib.b200_index_copy_rows(self.index._h, self.w0, m, self.buf.ctypes.data, None), "copy_rows")
            e = min(b, self.w1)
            out.append(self.buf[a - self.w0:e - self.w0])
            a = e


def write_index(index, path, chunk_bytes=1 << 26):
    """Write a built index as a FAISS index file, the file `load_index` (and clip back's faiss.read_index) opens.

        B200FlatIndex       -> IxSQ, QT_fp16
        B200IVFFlatIndex    -> IwSq, QT_fp16, by_residual = false
        B200IVFPQIndex      -> IwPQ (8-bit codes); with a pre-transform, inside one IxPT holding an LTra
        index_from_faiss's id-mapped wrapper -> IxMp around the above

    Rows are fp16 in this engine, so a flat or IVF-Flat index is always written as its SQfp16 form.  The coarse
    quantiser is always written as a flat IndexFlatIP (IxFI), also for an index built from an `_HNSW32` key: building
    an HNSW graph is out of scope, and FAISS then probes the centroids exactly, as this engine does.  IVF indices are
    finalized first.  The row / code store is streamed to the file `chunk_bytes` at a time (ids alike), so host memory
    stays bounded by the chunk, not by the index.  Refuses other objects and an index whose id_base is not 0.
    The layout restates FAISS's index_write.cpp and is UNVERIFIED against FAISS itself (see the module docstring)."""
    from ._lib import lib, check
    from .index import B200FlatIndex, B200IVFFlatIndex, B200IVFPQIndex, _IdMapped

    id_map = None
    inner = index
    if isinstance(index, _IdMapped):
        inner, id_map = index._index, index._map
    if not isinstance(inner, (B200FlatIndex, B200IVFFlatIndex, B200IVFPQIndex)):
        raise TypeError("write_index: %s is not an index of this engine (flat, IVF-Flat, IVF-PQ or an id-mapped one)"
                        % type(index).__name__)
    if inner.id_base != 0:
        raise ValueError("write_index: id_base=%d; a FAISS file numbers its rows from 0 (write each shard's index "
                         "before setting id_base, or wrap it in an id map)" % inner.id_base)
    if not isinstance(inner, B200FlatIndex):
        inner.finalize()
    info = np.zeros(8, np.int32)
    check(lib.b200_index_get_quantizer(inner._h, None, None, None, None, info.ctypes.data), "get_quantizer")
    nlist, M, by_residual, has_A, has_b, d, d_in, nprobe = (int(v) for v in info)
    n = inner.ntotal
    width = M if M else 2 * d
    chunk = max(1, chunk_bytes // width)
    with open(path, "wb") as f:
        out = _FileSink(f)
        if id_map is not None:
            _w_fourcc(out, "IxMp")
            _w_header(out, d_in, n, METRIC_INNER_PRODUCT)
        if nlist == 0:
            _w_fourcc(out, "IxSQ")
            _w_header(out, d, n, METRIC_INNER_PRODUCT)
            _w_sq_fp16(out, d)
            out.append(struct.pack("<Q", n * width))
            _StoreReader(inner, chunk, width, False).write(out, 0, n)
        else:
            cent = np.empty((nlist, d), np.float32)
            cb = np.empty((M, 256, d // M), np.float32) if M else None
            A = np.empty((d, d_in), np.float32) if has_A else None
            b = np.empty(d, np.float32) if has_b else None
            ptr = lambda a: None if a is None else a.ctypes.data  # noqa: E731
            check(lib.b200_index_get_quantizer(inner._h, ptr(cent), ptr(cb), ptr(A), ptr(b), None), "get_quantizer")
            if A is not None:
                _w_pretransform(out, A, b, n)
            if M:
                _w_ivf_head(out, "IwPQ", d, n, nprobe, cent)
                _w_ivfpq_params(out, d, M, by_residual, cb)
            else:
                _w_ivf_head(out, "IwSq", d, n, nprobe, cent)
                _w_sq_fp16(out, d)
                out.append(struct.pack("<QB", 2 * d, 0))
            sizes = np.zeros(nlist, np.int64)
            check(lib.b200_index_ivf_lists(inner._h, sizes.ctypes.data, None), "ivf_lists")
            _w_invlists_head(out, nlist, width, sizes)
            rows, ids = _StoreReader(inner, chunk, width, False), _StoreReader(inner, chunk, width, True)
            off = 0
            for m in sizes.tolist():
                if m:
                    rows.write(out, off, off + m)
                    ids.write(out, off, off + m)
                    off += m
        if id_map is not None:
            _w_vec(out, np.asarray(id_map, dtype=np.int64))
