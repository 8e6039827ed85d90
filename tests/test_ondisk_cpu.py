"""On-disk IVF-PQ files without a GPU: the ilod record (faiss_io.write_ivfpq_ondisk -> read_faiss_index), its
refusals, the in-place lists of ilar files, and index_combiner (FAISS merge_ondisk with shift_ids=False)."""
import os
import struct

import numpy as np
import pytest

import clip_retrieval_b200 as m
from clip_retrieval_b200 import faiss_io


def _quantiser(rng, d=32, M=8, nlist=6):
    C = rng.standard_normal((nlist, d)).astype(np.float32)
    cb = rng.standard_normal((M, 256, d // M)).astype(np.float32)
    return C, cb


def _rows(rng, n, M, nlist, empty=()):
    lists = rng.integers(0, nlist, n)
    for l in empty:
        lists[lists == l] = (l + 1) % nlist
    return rng.integers(0, 256, (n, M), dtype=np.uint8), lists


def _ilod_record(path):
    """The raw fields of the ilod record of `path`, parsed independently of faiss_io."""
    buf = open(path, "rb").read()
    at = buf.rindex(b"ilod") + 4
    nlist, code_size = struct.unpack_from("<QQ", buf, at)
    at += 16
    (nl,) = struct.unpack_from("<Q", buf, at)
    lists = np.frombuffer(buf, np.uint64, nl * 3, at + 8).reshape(-1, 3)
    at += 8 + 24 * nl
    (ns,) = struct.unpack_from("<Q", buf, at)
    slots = np.frombuffer(buf, np.uint64, ns * 2, at + 8).reshape(-1, 2)
    at += 8 + 16 * ns
    (nn,) = struct.unpack_from("<Q", buf, at)
    name = buf[at + 8:at + 8 + nn].decode()
    (totsize,) = struct.unpack_from("<Q", buf, at + 8 + nn)
    assert at + 16 + nn == len(buf)
    return nlist, code_size, lists.astype(np.int64), slots.astype(np.int64), name, totsize


def test_ilod_round_trip_and_record_bytes(tmp_path):
    rng = np.random.default_rng(1)
    M, nlist = 8, 6
    C, cb = _quantiser(rng, M=M, nlist=nlist)
    codes, lists = _rows(rng, 500, M, nlist, empty=(3,))
    ids = rng.permutation(10_000)[:500].astype(np.int64) + (1 << 33)
    spare = np.zeros(nlist, np.int64)
    spare[2] = 5                                   # capacity > size in list 2
    folder = str(tmp_path / "merged")
    triples = faiss_io.write_ivfpq_ondisk(folder, C, cb, codes, lists, ids=ids, nprobe=3, spare=spare,
                                          recorded_dir="/elsewhere/merge/run")
    nl, code_size, rec, slots, name, totsize = _ilod_record(os.path.join(folder, "populated.index"))
    sizes = np.bincount(lists, minlength=nlist)
    assert nl == nlist and code_size == M
    assert np.array_equal(rec, triples) and np.array_equal(rec[:, 0], sizes) and np.array_equal(rec[:, 1], sizes + spare)
    assert np.array_equal(rec[1:, 2], np.cumsum(rec[:, 1] * (M + 8))[:-1]) and rec[0, 2] == 0
    assert name == "/elsewhere/merge/run/merged_index.ivfdata"
    end = int((rec[:, 1] * (M + 8)).sum())
    assert slots.tolist() == [[end, 64]] and totsize == end + 64
    assert os.path.getsize(os.path.join(folder, "merged_index.ivfdata")) == totsize
    # the reader resolves the foreign path to the index's own folder (ONDISK_SAME_DIR)
    for target in (os.path.join(folder, "populated.index"),):
        r = faiss_io.read_faiss_index(target)
        inv = r["invlists"]
        assert r["kind"] == "ivfpq" and r["ntotal"] == 500 and r["nprobe"] == 3 and r["M"] == M
        assert np.array_equal(inv.id_off, rec[:, 2] + rec[:, 1] * M)        # id address: offset + capacity * code_size
        order = np.argsort(lists, kind="stable")
        assert np.array_equal(r["codes"], codes[order]) and np.array_equal(r["ids"], ids[order])
        for l in range(nlist):
            sel = order[np.isin(order, np.nonzero(lists == l)[0])]
            assert np.array_equal(inv.codes(l), codes[sel]) and np.array_equal(inv.ids(l), ids[sel])
            assert not inv.codes(l).flags.writeable and not inv.codes(l).flags.owndata     # views of the map
        code_addr, id_addr = inv.addresses()
        assert (id_addr - code_addr == (rec[:, 1] * M).astype(np.uint64)).all()


def test_ilar_lists_are_views_of_the_file(tmp_path):
    rng = np.random.default_rng(2)
    C, cb = _quantiser(rng)
    codes, lists = _rows(rng, 300, 8, 6, empty=(0, 4))
    p = str(tmp_path / "a.index")
    faiss_io.write_ivfpq(p, C, cb, codes, lists, ids=np.arange(300) * 3, sparse_sizes=True)
    r = faiss_io.read_faiss_index(p)
    inv = r["invlists"]
    assert inv.sizes[0] == 0 and inv.sizes[4] == 0
    raw = open(p, "rb").read()
    for l in np.nonzero(inv.sizes)[0]:
        c = inv.codes(l)
        assert not c.flags.owndata and raw[inv.code_off[l]:inv.code_off[l] + c.nbytes] == c.tobytes()
        assert inv.id_off[l] == inv.code_off[l] + c.nbytes


def _ondisk(tmp_path, **kw):
    rng = np.random.default_rng(3)
    C, cb = _quantiser(rng)
    codes, lists = _rows(rng, 200, 8, 6)
    folder = str(tmp_path / "f")
    t = faiss_io.write_ivfpq_ondisk(folder, C, cb, codes, lists, **kw)
    return folder, t


def test_ilod_refusals(tmp_path):
    folder, t = _ondisk(tmp_path / "ok")
    os.remove(os.path.join(folder, "merged_index.ivfdata"))
    with pytest.raises(ValueError, match="merged_index.ivfdata.*missing"):
        faiss_io.read_faiss_index(os.path.join(folder, "populated.index"))
    folder, t = _ondisk(tmp_path / "short", data_bytes=100)
    with pytest.raises(ValueError, match="short"):
        faiss_io.read_faiss_index(os.path.join(folder, "populated.index"))
    folder, t = _ondisk(tmp_path / "past")
    bad = t.copy()
    bad[4, 2] = 1 << 40
    faiss_io.write_ivfpq_ondisk(folder, *_quant_args(), lists_override=bad)
    with pytest.raises(ValueError, match="list 4 .*past the end"):
        faiss_io.read_faiss_index(os.path.join(folder, "populated.index"))
    bad = t.copy()
    bad[2, 1] = bad[2, 0] - 1
    faiss_io.write_ivfpq_ondisk(folder, *_quant_args(), lists_override=bad)
    with pytest.raises(ValueError, match="list 2 has capacity"):
        faiss_io.read_faiss_index(os.path.join(folder, "populated.index"))
    faiss_io.write_ivfpq_ondisk(folder, *_quant_args(), code_size=9)
    with pytest.raises(ValueError, match="code size 9"):
        faiss_io.read_faiss_index(os.path.join(folder, "populated.index"))


def _quant_args():
    rng = np.random.default_rng(3)
    C, cb = _quantiser(rng)
    codes, lists = _rows(rng, 200, 8, 6)
    return C, cb, codes, lists


def _parts(tmp_path, nparts, rng, C, cb, n_each=150, transform=None, hnsw=False):
    src = tmp_path / "parts"
    src.mkdir()
    allc, alll, alli = [], [], []
    for i in range(nparts):
        codes, lists = _rows(rng, n_each, cb.shape[0], C.shape[0], empty=((i,) if i < C.shape[0] else ()))
        ids = np.arange(i * n_each, (i + 1) * n_each, dtype=np.int64)   # global ids, as add_with_ids stores them
        faiss_io.write_ivfpq(str(src / ("block_%02d.index" % i)), C, cb, codes, lists, ids=ids, nprobe=2,
                             transform=transform, hnsw=hnsw)
        allc.append(codes)
        alll.append(lists)
        alli.append(ids)
    (src / "notes.txt").write_text("not a part")
    return str(src), allc, alll, alli


@pytest.mark.parametrize("nparts", [1, 3])
def test_index_combiner_concatenates_lists_in_file_order(tmp_path, nparts):
    rng = np.random.default_rng(4 + nparts)
    C, cb = _quantiser(rng)
    A = np.linalg.qr(rng.standard_normal((32, 32)))[0].astype(np.float32)
    src, allc, alll, alli = _parts(tmp_path, nparts, rng, C, cb, transform=(A, None), hnsw=True)
    out = str(tmp_path / "merged")
    m.index_combiner(src, out)
    assert sorted(os.listdir(out)) == ["merged_index.ivfdata", "populated.index"]
    r = faiss_io.read_faiss_index(os.path.join(out, "populated.index"))
    assert r["ntotal"] == nparts * 150 and r["nprobe"] == 2 and np.array_equal(r["transform"][0], A)
    raw = open(os.path.join(out, "populated.index"), "rb").read()
    assert struct.unpack_from("<q", raw, 8)[0] == nparts * 150          # IxPT header ntotal
    nl, code_size, rec, slots, name, totsize = _ilod_record(os.path.join(out, "populated.index"))
    assert np.array_equal(rec[:, 0], rec[:, 1]) and slots.size == 0 and code_size == 8
    assert np.array_equal(rec[:, 2], np.concatenate([[0], np.cumsum(rec[:, 1] * 16)[:-1]]))
    assert os.path.basename(name) == "merged_index.ivfdata" and totsize == os.path.getsize(os.path.join(out, name))
    inv = r["invlists"]
    for l in range(C.shape[0]):
        want_c = np.concatenate([c[ls == l] for c, ls in zip(allc, alll)])
        want_i = np.concatenate([i[ls == l] for i, ls in zip(alli, alll)])
        assert np.array_equal(inv.codes(l), want_c) and np.array_equal(inv.ids(l), want_i)
    if nparts == 3:
        assert (inv.sizes == 0).sum() == 0 and min(inv.sizes) >= 1   # lists empty in one part are filled by others


def test_index_combiner_refusals(tmp_path):
    rng = np.random.default_rng(9)
    C, cb = _quantiser(rng)
    A = np.linalg.qr(rng.standard_normal((32, 32)))[0].astype(np.float32)
    codes, lists = _rows(rng, 100, 8, 6)
    for what, kw in (("centroids", dict(C=C + 1)), ("codebook", dict(cb=cb * 2)),
                     ("pre-transform", dict(transform=(A[::-1].copy(), None)))):
        src = tmp_path / what
        src.mkdir()
        faiss_io.write_ivfpq(str(src / "a.index"), C, cb, codes, lists, transform=(A, None))
        faiss_io.write_ivfpq(str(src / "b.index"), kw.get("C", C), kw.get("cb", cb), codes, lists,
                             transform=kw.get("transform", (A, None)))
        with pytest.raises(ValueError, match="b.index differs .* in its " + what):
            m.index_combiner(str(src), str(tmp_path / ("out_" + what)))
    src = tmp_path / "idmap"
    src.mkdir()
    faiss_io.write_ivfpq(str(src / "a.index"), C, cb, codes, lists, id_map=np.arange(100) + 5)
    with pytest.raises(ValueError, match="id map"):
        m.index_combiner(str(src), str(tmp_path / "out_idmap"))
    (tmp_path / "empty").mkdir()
    with pytest.raises(ValueError, match="no file"):
        m.index_combiner(str(tmp_path / "empty"), str(tmp_path / "x"))
