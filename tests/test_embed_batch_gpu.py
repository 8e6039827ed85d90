"""Parity of the embed path ON THE KERNELS THE BENCH TIMES: batches large enough that every per-layer GEMM
takes the 128x128-tile wgmma kernel over the whole grid (gemm_pick_bn: >= 132 tiles) including the patch-embed epilogue
(row remap past the cls slot + positional residual) and the in-place residual epilogues, and the pipelined
host entry (four sub-batch slots, copy/compute streams) with batches larger than max_batch.
Tolerance: north_star's 1e-3 cosine against the fp32 oracle."""
import os

import numpy as np
import pytest

from oracle import clip_ref

pytestmark = pytest.mark.gpu
COS_TOL = 1e-3


def _arch(m, cfg):
    return m.ClipArch(cfg.embed_dim, cfg.image_size, cfg.patch,
                      m.Tower(cfg.vision.width, cfg.vision.layers, cfg.vision.heads, cfg.vision.mlp),
                      m.Tower(cfg.text.width, cfg.text.layers, cfg.text.heads, cfg.text.mlp),
                      cfg.context_length, cfg.vocab_size, cfg.quick_gelu)


def _tiles(M, N):
    return ((M + 127) // 128) * ((N + 127) // 128)


@pytest.fixture(scope="module")
def l14():
    import torch
    import clip_retrieval_b200 as m

    torch.set_num_threads(max(1, os.cpu_count() or 1))
    cfg = clip_ref.CONFIGS["ViT-L/14"]
    sd = clip_ref.make_state_dict(cfg, seed=0)
    model = m.B200Clip(_arch(m, cfg), device=0, max_batch=256)
    model.load_state_dict(sd)
    return model, cfg, sd


@pytest.mark.timeout(900)
def test_vit_l14_image_batch48_pair_gemm_matches_oracle(l14):
    """B=48: 97 row blocks x 8 column blocks = 776 tiles for out-proj (N=1024), 768 for the patch GEMM."""
    model, cfg, sd = l14
    B = 48
    assert _tiles(B * 257, 1024) >= 132 and _tiles(B * 256, 1024) >= 132
    px = clip_ref.synth_images(B, cfg, seed=11)
    got = model.embed_image_device(px.cuda()).cpu().numpy()
    ref = clip_ref.mapper_image(sd, cfg, px)
    c = 1 - clip_ref.cosine(got, ref)
    assert np.isfinite(got.astype(np.float32)).all()
    assert c.max() <= COS_TOL, c


@pytest.mark.timeout(900)
def test_vit_l14_text_batch192_pair_gemm_matches_oracle(l14):
    """B=192: 116 row blocks x 6 column blocks = 696 tiles for out-proj / c_proj (N=768)."""
    model, cfg, sd = l14
    B = 192
    assert _tiles(B * 77, 768) >= 132
    tk = clip_ref.synth_tokens(B, cfg, seed=12)
    got = model.embed_text_device(tk.cuda()).cpu().numpy()
    ref = clip_ref.mapper_text(sd, cfg, tk)
    c = 1 - clip_ref.cosine(got, ref)
    assert np.isfinite(got.astype(np.float32)).all()
    assert c.max() <= COS_TOL, c


@pytest.mark.timeout(600)
def test_pair_and_single_cta_gemm_agree_inside_the_model_at_batch_1024():
    """The bench configuration (ViT-L/14, batch 1024: 128-column tiles) against the same samples at batch 4, where
    every GEMM takes the narrow 32 / 64-column tiles of the serving shapes: both run the same K order with fp32
    accumulation, so the embeddings agree to the last bf16 rounding of the towers."""
    import torch
    import clip_retrieval_b200 as m

    arch = m.ARCHS["ViT-L/14"]
    model = m.B200Clip(arch, device=0, max_batch=1024)
    model.load_state_dict(m.synthetic_state_dict(arch, seed=0))
    g = torch.Generator().manual_seed(5)
    px = torch.randn(1024, 3, 224, 224, generator=g).clamp_(-1.80, 2.15).cuda()
    cfg = clip_ref.CONFIGS["ViT-L/14"]
    tk = clip_ref.synth_tokens(1024, cfg, seed=5).cuda()
    a_i, a_t = model.embed_image_device(px).float().cpu().numpy(), model.embed_text_device(tk).float().cpu().numpy()
    few = [0, 1, 2, 3]
    b_i, b_t = model.embed_image_device(px[few]).float().cpu().numpy(), model.embed_text_device(tk[few]).float().cpu().numpy()
    a_i4, a_t4 = a_i[few], a_t[few]
    for a, b in ((a_i4, b_i), (a_t4, b_t)):
        assert np.isfinite(a).all() and np.isfinite(b).all()
        assert (1 - clip_ref.cosine(a, b)).max() <= 2e-5
        assert np.abs(a - b).max() <= 4e-3   # a few fp16/bf16 ulps of unit-norm components
    assert np.isfinite(a_i).all() and np.isfinite(a_t).all()
    # and the batch-1024 result agrees with the oracle on a handful of samples spread over the batch
    sel = [0, 511, 1023]
    sd = {k: v for k, v in m.synthetic_state_dict(arch, seed=0).items()}
    ref_i = clip_ref.mapper_image(sd, cfg, px[sel].cpu())
    ref_t = clip_ref.mapper_text(sd, cfg, tk[sel].cpu())
    assert (1 - clip_ref.cosine(a_i[sel], ref_i)).max() <= COS_TOL
    assert (1 - clip_ref.cosine(a_t[sel], ref_t)).max() <= COS_TOL


@pytest.mark.timeout(600)
@pytest.mark.parametrize("B", [600])
def test_pipelined_host_entry_matches_device_entry(B):
    """encode_host with max_batch >= 256 splits images into four sub-batch slots (H2D on the copy stream
    overlapping compute) and loops over chunks of max_batch; B = 600 = 256 + 256 + 88 leaves a ragged last
    chunk (64 + 24).  Per-sample results must not depend on the slot they travelled through."""
    import torch
    import clip_retrieval_b200 as m

    cfg = clip_ref.CONFIGS["ViT-B/32"]
    sd = clip_ref.make_state_dict(cfg, seed=0)
    model = m.B200Clip(_arch(m, cfg), device=0, max_batch=256)
    model.load_state_dict(sd)
    px = clip_ref.synth_images(B, cfg, seed=21)
    tk = clip_ref.synth_tokens(B, cfg, seed=21)
    hi, ht = model.embed_image(px), model.embed_text(tk)           # host buffers, pipelined
    hi2 = model.embed_image(px.pin_memory())                       # pinned source, second pass over the slot ring
    assert hi.shape == (B, cfg.embed_dim) and hi.dtype == np.float16 and np.array_equal(hi, hi2)
    di = np.concatenate([model.embed_image_device(px[i:i + 32].cuda()).cpu().numpy() for i in range(0, B, 32)])
    dt = np.concatenate([model.embed_text_device(tk[i:i + 32].cuda()).cpu().numpy() for i in range(0, B, 32)])
    assert np.isfinite(hi.astype(np.float32)).all() and np.isfinite(ht.astype(np.float32)).all()
    assert (1 - clip_ref.cosine(hi, di)).max() <= 1e-5 and np.abs(hi.astype(np.float32) - di.astype(np.float32)).max() <= 2e-3
    assert (1 - clip_ref.cosine(ht, dt)).max() <= 1e-5
    sel = sorted(set([0, 63, 64, 255, 256, B - 1]) & set(range(B)))
    assert (1 - clip_ref.cosine(hi[sel], clip_ref.mapper_image(sd, cfg, px[sel]))).max() <= COS_TOL
    assert (1 - clip_ref.cosine(ht[sel], clip_ref.mapper_text(sd, cfg, tk[sel]))).max() <= COS_TOL


@pytest.mark.timeout(300)
def test_concurrent_host_and_device_encodes_share_one_handle_safely():
    """clip_back serves from Flask threads (clip_back.py:1018): host-entry and device-entry forwards on one
    handle from two threads / two streams must each return what they return alone."""
    import threading

    import torch
    import clip_retrieval_b200 as m

    cfg = clip_ref.CONFIGS["tiny"]
    sd = clip_ref.make_state_dict(cfg, seed=0)
    model = m.B200Clip(_arch(m, cfg), device=0, max_batch=8)
    model.load_state_dict(sd)
    px = clip_ref.synth_images(8, cfg, seed=3)
    tk = clip_ref.synth_tokens(8, cfg, seed=3)
    want_i, want_t = model.embed_image(px), model.embed_text(tk)
    errs = []

    def host_worker():
        for _ in range(40):
            if not np.array_equal(model.embed_image(px), want_i):
                errs.append("host image")

    def device_worker():
        s = torch.cuda.Stream()
        tkd = tk.cuda()
        with torch.cuda.stream(s):
            for _ in range(40):
                out = model.embed_text_device(tkd)
                s.synchronize()
                if not np.array_equal(out.cpu().numpy(), want_t):
                    errs.append("device text")

    ts = [threading.Thread(target=host_worker), threading.Thread(target=device_worker)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert not errs, errs[:4]
