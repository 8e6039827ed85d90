"""wgmma GEMM core vs a plain fp32 PyTorch reference of the same op (floating-point kernel:
tolerance = bf16 output rounding 2^-8 relative + accumulation noise, stated per assert)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _ref(A, W, b, R, act):
    import torch

    ref = A.float() @ W.float().t()
    if b is not None:
        ref = ref + b
    if act == 1:
        ref = ref * torch.sigmoid(1.702 * ref)
    elif act == 2:
        ref = torch.nn.functional.gelu(ref)
    if R is not None:
        ref = ref + R.float()
    return ref


@pytest.mark.timeout(120)
@pytest.mark.parametrize(
    "M,N,K,act,bias,res",
    [
        (128, 256, 64, 0, False, False),
        (1, 512, 512, 0, True, False),        # single row (B=1 serving shape)
        (257, 768, 768, 1, True, True),       # ragged M
        (77 * 3, 2304, 768, 0, True, False),  # text QKV
        (1000, 3072, 1024, 2, True, True),
        (300, 1280, 1280, 0, True, True),     # H/14 width: 128-wide column blocks
        (130, 520, 328, 1, True, True),       # N, K not multiples of the tile: TMA zero fill + predication
        (4112, 4096, 1024, 1, True, False),
        (4112, 1024, 4096, 0, True, True),
        (20001, 3072, 1024, 1, True, True),   # CTA-pair kernel (256x256 tiles), ragged M
        (19000, 1000, 520, 2, True, True),    # CTA-pair kernel, N and K tails
    ],
)
def test_gemm_matches_fp32_reference(M, N, K, act, bias, res):
    import torch
    from clip_retrieval_b200._lib import lib, check

    g = torch.Generator(device="cuda").manual_seed(M + 31 * N + 977 * K)
    A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).bfloat16()
    W = (torch.randn(N, K, device="cuda", generator=g) * 0.05).bfloat16()
    b = torch.randn(N, device="cuda", generator=g) if bias else None
    R = torch.randn(M, N, device="cuda", generator=g).bfloat16() if res else None
    out = torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
    st = torch.cuda.current_stream().cuda_stream
    check(lib.b200_gemm_bf16_device(A.data_ptr(), W.data_ptr(), b.data_ptr() if bias else None,
                                    R.data_ptr() if res else None, out.data_ptr(), M, N, K, act, 0, st), "gemm")
    torch.cuda.synchronize()
    ref = _ref(A, W, b, R, act)
    err = (out.float() - ref).abs()
    # bf16 output: half an ulp = 2^-9 relative; allow 2^-7 relative + 0.02 absolute for the fp32 sums
    assert not torch.isnan(out.float()).any()
    assert bool((err <= ref.abs() * 2 ** -7 + 0.02).all()), "max err %g" % err.max().item()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("M,N,K,act,bias,res", [
    (20001, 3072, 1024, 1, True, False),   # qkv / fc shape class, ragged M
    (20001, 1024, 1024, 0, True, True),    # out-proj: residual stored in place of it
    (19000, 1000, 520, 2, True, True),     # N and K tails: boxes clipped by the tensor maps
    (40000, 768, 3072, 0, True, True),     # text c_proj shape class
    (20001, 512, 1024, 0, True, False),    # plain bias epilogue (qkv)
    (20001, 1024, 1024, 1, True, True),    # QuickGELU + residual
    (20001, 1024, 512, 2, False, False),   # erf-GELU, no bias
])
def test_pair_gemm_tma_store_equals_register_store(M, N, K, act, bias, res):
    """Full-grid shapes with every epilogue flavour (activation, bias, residual): the result stored into a fresh buffer
    and the result stored over its own residual (in-place update of the residual stream, as the model runs it) are
    bit-identical, and both match the fp32 reference."""
    import torch
    from clip_retrieval_b200._lib import lib, check

    g = torch.Generator(device="cuda").manual_seed(M + 31 * N + 977 * K)
    A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).bfloat16()
    W = (torch.randn(N, K, device="cuda", generator=g) * 0.05).bfloat16()
    b = torch.randn(N, device="cuda", generator=g) if bias else None
    R = torch.randn(M, N, device="cuda", generator=g).bfloat16() if res else None
    st = torch.cuda.current_stream().cuda_stream
    outs = []
    for in_place in (False, True):
        out = R.clone() if (res and in_place) else torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
        check(lib.b200_gemm_bf16_device(A.data_ptr(), W.data_ptr(), b.data_ptr() if bias else None,
                                        (out if in_place else R).data_ptr() if res else None, out.data_ptr(), M, N, K, act, 0,
                                        st), "gemm")
        torch.cuda.synchronize()
        outs.append(out)
    assert not torch.isnan(outs[0].float()).any()
    assert torch.equal(outs[0], outs[1]), "in-place vs separate output: max diff %g" % (outs[0].float() - outs[1].float()).abs().max().item()
    ref = _ref(A, W, b, R, act)
    err = (outs[0].float() - ref).abs()
    assert bool((err <= ref.abs() * 2 ** -7 + 0.02).all()), "max err %g" % err.max().item()


@pytest.mark.timeout(300)
def test_run_time_epilogue_with_folded_layernorm_matches_oracle():
    """The run-time epilogue flavour (every feature decided per launch: LayerNorm folded into the qkv / fc GEMMs, row
    statistics written by the residual GEMMs), reached through B200_FUSE_LN=1: ViT-B/32 embeddings against the
    fp32 oracle and against the default path (separate LayerNorm kernel, compile-time epilogue flavours)."""
    import os

    import clip_retrieval_b200 as m
    from oracle import clip_ref

    cfg = clip_ref.CONFIGS["ViT-B/32"]
    sd = clip_ref.make_state_dict(cfg, seed=0)
    arch = m.ClipArch(cfg.embed_dim, cfg.image_size, cfg.patch,
                      m.Tower(cfg.vision.width, cfg.vision.layers, cfg.vision.heads, cfg.vision.mlp),
                      m.Tower(cfg.text.width, cfg.text.layers, cfg.text.heads, cfg.text.mlp),
                      cfg.context_length, cfg.vocab_size, cfg.quick_gelu)
    px, tk = clip_ref.synth_images(6, cfg, seed=4), clip_ref.synth_tokens(6, cfg, seed=4)
    outs = {}
    old = os.environ.get("B200_FUSE_LN")
    try:
        for fuse in ("0", "1"):
            os.environ["B200_FUSE_LN"] = fuse
            model = m.B200Clip(arch, device=0, max_batch=8).load_state_dict(sd)
            outs[fuse] = (model.embed_image(px), model.embed_text(tk))
            del model
    finally:
        if old is None:
            os.environ.pop("B200_FUSE_LN", None)
        else:
            os.environ["B200_FUSE_LN"] = old
    ref_i, ref_t = clip_ref.mapper_image(sd, cfg, px), clip_ref.mapper_text(sd, cfg, tk)
    for (ei, et) in outs.values():
        assert np.isfinite(ei.astype(np.float32)).all() and np.isfinite(et.astype(np.float32)).all()
        assert (1 - clip_ref.cosine(ei, ref_i)).max() <= 1e-3 and (1 - clip_ref.cosine(et, ref_t)).max() <= 1e-3
    assert (1 - clip_ref.cosine(outs["1"][0], outs["0"][0])).max() <= 1e-3
    assert (1 - clip_ref.cosine(outs["1"][1], outs["0"][1])).max() <= 1e-3
