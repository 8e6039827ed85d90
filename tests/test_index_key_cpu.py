"""The index factory strings clip_index builds, and this project's default key rule at its boundaries."""
import math

import pytest

import clip_retrieval_b200 as m
from clip_retrieval_b200.clip_index import memory_bytes


@pytest.mark.parametrize("key,kind,nlist,M,opq_M,opq_dim,hnsw", [
    ("SQfp16", "flat", 0, 0, 0, 0, 0),
    ("Flat", "flat", 0, 0, 0, 0, 0),
    ("IVF1024,Flat", "ivfflat", 1024, 0, 0, 0, 0),
    ("IVF7,SQfp16", "ivfflat", 7, 0, 0, 0, 0),
    ("IVF4096,PQ64x8", "ivfpq", 4096, 64, 0, 0, 0),
    ("IVF4096_HNSW32,PQ64x8", "ivfpq", 4096, 64, 0, 0, 32),
    ("OPQ64_768,IVF4096_HNSW32,PQ64x8", "ivfpq", 4096, 64, 64, 768, 32),
    ("OPQ16_64,IVF256,PQ16x8", "ivfpq", 256, 16, 16, 64, 0),
    ("OPQ32,IVF256,PQ32x8", "ivfpq", 256, 32, 32, 0, 0),
])
def test_accepted_forms(key, kind, nlist, M, opq_M, opq_dim, hnsw):
    k = m.parse_index_key(key)
    assert (k.kind, k.nlist, k.M, k.opq_M, k.opq_dim, k.hnsw) == (kind, nlist, M, opq_M, opq_dim, hnsw)


@pytest.mark.parametrize("key,component", [
    ("HNSW32", "HNSW32"),
    ("PCA64,IVF100,Flat", "PCA64"),
    ("IVF100,PQ16x4", "PQ16x4"),
    ("IVF100,PQ16x4fs", "PQ16x4fs"),
    ("IVF100,SQ8", "SQ8"),
    ("IVF100,Flat,RFlat", "RFlat"),
    ("OPQ16_64,IVF100,Flat", "OPQ16_64,IVF100,Flat"),
    ("PQ16x8", "PQ16x8"),
    ("IVF100_HNSW32,Flat", "IVF100_HNSW32,Flat"),
    ("IVF100", "IVF100"),
    ("OPQ16,PQ16x8", "OPQ16,PQ16x8"),
])
def test_refused_forms_name_the_component(key, component):
    with pytest.raises(NotImplementedError, match=component):
        m.parse_index_key(key)


def test_memory_sizes():
    assert memory_bytes("4G") == 4 << 30 and memory_bytes("16GB") == 16 << 30 and memory_bytes("512M") == 512 << 20
    assert memory_bytes(1000) == 1000 and memory_bytes("1.5K") == 1536
    with pytest.raises(ValueError):
        memory_bytes("lots")


def test_default_key_boundaries():
    G = 1 << 30
    assert m.default_index_key(9999, 768, "1K") == "SQfp16"
    n = 10000
    nlist = 2 ** round(math.log2(4 * math.sqrt(n)))
    assert nlist == 512
    assert m.default_index_key(n, 768, n * (2 * 768 + 8)) == "IVF512,SQfp16"
    assert m.default_index_key(n, 768, n * (2 * 768 + 8) - 1) == "OPQ256_768,IVF512_HNSW32,PQ256x8"
    assert m.default_index_key(n, 768, n * (256 + 8) - 1) == "OPQ128_768,IVF512_HNSW32,PQ128x8"
    assert m.default_index_key(n, 768, n * (8 + 8)) == "OPQ8_768,IVF512_HNSW32,PQ8x8"
    with pytest.raises(ValueError, match=str(n * 16)):
        m.default_index_key(n, 768, n * 16 - 1)
    # d = 96: 256 and 128 do not divide it, 32 is the largest that does
    assert m.default_index_key(n, 96, n * (32 + 8)) == "OPQ32_96,IVF512_HNSW32,PQ32x8"
    # nlist: 2^round(log2(4 sqrt(N))) on both sides of a rounding boundary (4 sqrt(N) = 2^9.5 at N = 32768)
    assert m.default_index_key(32767, 64, 4 * G) == "IVF512,SQfp16"
    assert m.default_index_key(32769, 64, 4 * G) == "IVF1024,SQfp16"
    with pytest.raises(ValueError):
        m.default_index_key(10 ** 9, 768, "4G")


def test_default_nprobe():
    assert [m.default_nprobe(n) for n in (1, 3, 4, 512, 4096, 65536)] == [1, 1, 2, 22, 64, 256]
