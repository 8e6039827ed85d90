"""Sharded search on hardware (SURVEY.md §8e): the packed candidate block + in-place merge used around the one
all-gather, the single-process peer-memory exchange behind the C ABI (`b200_sharded_search`), and the
one-process-per-GPU NCCL path.  Multi-device cases skip on a one-GPU box (the driver's `-m gpu` run); they run
under `gpurun --gpus 2`."""
import os
import sys

import numpy as np
import pytest

from oracle import knn_ref, synth_ref

pytestmark = pytest.mark.gpu
TOL = 2e-6
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ngpu():
    import torch

    return torch.cuda.device_count()


@pytest.mark.parametrize("G,nq,k", [(2, 1, 40), (4, 5, 40), (8, 33, 7), (3, 1000, 40)])
def test_packed_blocks_merge_in_place(G, nq, k):
    """Every shard's search writes (I, D) into its slot of one buffer (what the all-gather delivers); the merge
    reads that buffer in place.  Result == merge of the same candidates by the oracle == single-index search."""
    import torch
    import clip_retrieval_b200 as m
    from clip_retrieval_b200.sharded import block_bytes

    d, n = 256, 9000
    X = synth_ref.rows_f16(n, d)
    Q = synth_ref.rows_f32(nq, d, seed=4321)
    qd = torch.from_numpy(Q).cuda()
    blk = block_bytes(nq, k)
    recv = torch.zeros(G * blk, dtype=torch.uint8, device="cuda")
    Dg, Ig = [], []
    for g in range(G):
        lo, hi = m.shard_range(n, G, g)
        idx = m.B200FlatIndex(d)
        idx.add(X[lo:hi])
        idx.id_base = lo
        slot = recv[g * blk:(g + 1) * blk]
        I = slot[:nq * k * 8].view(torch.int64).view(nq, k)
        D = slot[nq * k * 8:nq * k * 12].view(torch.float32).view(nq, k)
        idx.search_device(qd, k, out=(D, I))
        Dg.append(D.cpu().numpy().copy())
        Ig.append(I.cpu().numpy().copy())
    D, I = m.merge_packed_results(recv, G, blk, nq, k)
    Do, Io = knn_ref.merge_shards(np.stack(Dg), np.stack(Ig), k)
    assert np.array_equal(I.cpu().numpy(), Io) and np.array_equal(D.cpu().numpy(), Do)   # pure selection: exact
    ok, msg, _ = knn_ref.check_topk(D.cpu().numpy(), I.cpu().numpy(), knn_ref.scores_f64(X, Q), k, tol=TOL)
    assert ok, msg


def test_sharded_ivf_equals_single_ivf():
    """IVF-Flat shards built over the replicated global centroids: the union over shards of list l is the global
    list l, so with equal nprobe the merged result is identical to the single-index result (SURVEY §8e)."""
    import torch
    import clip_retrieval_b200 as m
    from clip_retrieval_b200.sharded import block_bytes

    d, n, nlist, k, nq, G = 128, 40000, 64, 40, 9, 4
    kw = dict(seed=5, clustered=True, centroid_seed=7, nlist=nlist, cw=3, nw=1)
    spec = m.SynthSpec(**kw)
    X = synth_ref.rows_f16(n, d, **kw)
    C = synth_ref.centroids_f32(nlist, d, 7)
    Q = synth_ref.rows_f32(nq, d, seed=77, clustered=True, centroid_seed=7, nlist=nlist)
    qd = torch.from_numpy(Q).cuda()
    for nprobe in (1, 4, 64):
        whole = m.B200IVFFlatIndex(d, nlist, C)
        whole.add(X)
        whole.nprobe = nprobe
        Dw, Iw = whole.search_device(qd, k)
        blk = block_bytes(nq, k)
        recv = torch.zeros(G * blk, dtype=torch.uint8, device="cuda")
        for g in range(G):
            lo, hi = m.shard_range(n, G, g)
            sh = m.B200IVFFlatIndex(d, nlist, C)
            if g % 2 == 0:
                sh.add(X[lo:hi])
            else:
                sh.add_synthetic(hi - lo, spec, row0=lo)     # rows generated on the device, general bucketing path
            sh.id_base = lo
            sh.nprobe = nprobe
            slot = recv[g * blk:(g + 1) * blk]
            sh.search_device(qd, k, out=(slot[nq * k * 8:nq * k * 12].view(torch.float32).view(nq, k),
                                         slot[:nq * k * 8].view(torch.int64).view(nq, k)))
        D, I = m.merge_packed_results(recv, G, blk, nq, k)
        assert torch.equal(I, Iw) and torch.equal(D, Dw), "nprobe=%d" % nprobe
        # and against the CPU oracle's IVF search
        assign = knn_ref.ivf_assign(X, C.astype(np.float16))
        Do, Io, _ = knn_ref.ivf_search(X, assign, C.astype(np.float16), Q, k, nprobe)
        np.testing.assert_allclose(D.cpu().numpy(), Do, atol=TOL)
        assert (I.cpu().numpy() == Io).mean() > 0.995


@pytest.mark.parametrize("use_nccl", [False, True])
def test_single_process_sharded_search_c_abi(use_nccl):
    """b200_sharded_search: one host call over every GPU of the box; candidates reach the root as peer stores
    from the search epilogue (or through one ncclAllGather group)."""
    if _ngpu() < 2:
        pytest.skip("needs >= 2 GPUs")
    import clip_retrieval_b200 as m

    G = min(_ngpu(), 8)
    d, n, k = 768, 60000, 40
    X = synth_ref.rows_f16(n, d)
    shards = []
    for g in range(G):
        lo, hi = m.shard_range(n, G, g)
        idx = m.B200FlatIndex(d, device=g)
        idx.add(X[lo:hi])
        idx.id_base = lo
        shards.append(idx)
    sh = m.B200ShardedIndex(shards, use_nccl=use_nccl)
    for nq in (1, 7, 300):
        Q = synth_ref.rows_f32(nq, d, seed=4321 + nq)
        D, I = sh.search(Q, k)
        ok, msg, strict = knn_ref.check_topk(D, I, knn_ref.scores_f64(X, Q), k, tol=TOL)
        assert ok, msg
        D2, I2 = sh.search(Q, k)
        assert np.array_equal(I, I2) and np.array_equal(D, D2)
    if not use_nccl:
        assert sh.peer_mode, "NVSwitch boxes map every peer"


def _nccl_worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch
    import torch.distributed as dist

    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    import clip_retrieval_b200 as m

    n, d, k = 50003, 768, 40
    lo, hi = m.shard_range(n, world, rank)
    idx = m.B200FlatIndex(d, device=rank)
    idx.add_synthetic(hi - lo, m.SynthSpec(seed=3), row0=lo)
    idx.id_base = lo
    sh = m.ShardedIndex(idx, device=torch.device("cuda", rank))
    out = {}
    for nq in (1, 64, 1000):
        Q = synth_ref.rows_f32(nq, d, seed=8 + nq)
        D, I = sh.search(Q, k)
        Dg, Ig = sh.gathered_candidates()
        out["D%d" % nq], out["I%d" % nq], out["Dg%d" % nq], out["Ig%d" % nq] = D, I, Dg, Ig
    np.savez(os.path.join(out_dir, "r%d.npz" % rank), **out)
    dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_nccl_sharded_search_equals_single_index(tmp_path):
    """One process per GPU, NCCL all-gather of the packed blocks, merge in place — checked on hardware against the
    oracle's merge of the gathered candidates (bit-exact) and the float64 ranking of the whole index."""
    if _ngpu() < 2:
        pytest.skip("needs >= 2 GPUs")
    import torch.multiprocessing as mp

    world, port = 2, 29700 + os.getpid() % 2000
    mp.spawn(_nccl_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    X = synth_ref.rows_f16(50003, 768, seed=3)
    for nq in (1, 64, 1000):
        Q = synth_ref.rows_f32(nq, 768, seed=8 + nq)
        got = [np.load(os.path.join(str(tmp_path), "r%d.npz" % r)) for r in range(world)]
        for r in range(world):
            assert np.array_equal(got[r]["I%d" % nq], got[0]["I%d" % nq]) and np.array_equal(got[r]["D%d" % nq], got[0]["D%d" % nq])
            Do, Io = knn_ref.merge_shards(got[r]["Dg%d" % nq], got[r]["Ig%d" % nq], 40)
            assert np.array_equal(got[r]["I%d" % nq], Io) and np.array_equal(got[r]["D%d" % nq], Do)
        ok, msg, _ = knn_ref.check_topk(got[0]["D%d" % nq], got[0]["I%d" % nq], knn_ref.scores_f64(X, Q), 40, tol=TOL)
        assert ok, msg
