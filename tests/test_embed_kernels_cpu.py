"""The bounds of test_embed_kernels_gpu.py can fail: for each one, float64 computations of plausible wrong kernels on the
same kind of inputs, stored as the kernel stores, break it on at least one element, while the right operation computed
in fp32 and stored the same way stays inside it.  And every entry of the model tables maps to a kernel case."""
import math

import pytest
import torch

import embed_kernels_ref as R

LN_WIDTHS = sorted(set(R.LN_TEMPLATE_WIDTHS) | {w for w, _ in R.layernorm_cases()})


def _ln_fp32(x, ga, be, eps):
    """A right LayerNorm in fp32 arithmetic (torch's summation order), stored as bf16."""
    xf = x.float()
    mu = xf.mean(-1, keepdim=True)
    d = xf - mu
    return (d * torch.rsqrt((d * d).mean(-1, keepdim=True) + eps) * ga + be).bfloat16()


@pytest.mark.parametrize("eps", R.LN_EPS)
@pytest.mark.parametrize("w", LN_WIDTHS)
def test_layernorm_bound_rejects_wrong_kernels(w, eps):
    x, ga, be, cls = R.layernorm_inputs(200, w, seed=w, device="cpu")
    ref, bound = R.layernorm_bound(x, ga, be, eps, "rows")
    assert R.within(ref.bfloat16(), ref, bound)
    assert R.within(_ln_fp32(x, ga, be, eps), ref, bound)
    live = cls != 4          # constant rows: every variant but the eps-free one gives beta there too

    def rejected(y):
        return not R.within(y.bfloat16()[live], ref[live], bound[live])

    variants = {
        "variance / (w - 1)": R.layernorm_bound(x, ga, be, eps, "rows", variance_divisor=w - 1)[0],
        "eps x 10": R.layernorm_bound(x, ga, be, 10 * eps, "rows")[0],
        "eps dropped": R.layernorm_bound(x, ga, be, 0.0, "rows")[0],
    }
    if w > 256:
        # a kernel that reduces only the first 32 lanes x 8 columns for the mean (the variance still over the row)
        xd = x.double()
        mu = xd[:, :256].mean(-1, keepdim=True)
        d = xd - mu
        variants["mean of the first 256 columns"] = d * ((d * d).mean(-1, keepdim=True) + eps).rsqrt() * ga.double() \
            + be.double()
    for name, y in variants.items():
        assert rejected(y), "w=%d eps=%g: the bound accepts the LayerNorm with %s" % (w, eps, name)


def _pool_inputs(B, T, w, D, seed):
    g = torch.Generator().manual_seed(seed)
    x, ga, be, _ = R.layernorm_inputs(B * T, w, seed, "cpu")
    proj = (torch.randn(w, D, generator=g) * w ** -0.5).bfloat16()
    return x.view(B, T, w), ga, be, proj


@pytest.mark.parametrize("w,D,T", R.pool_cases())
def test_pool_ln_proj_bound_rejects_wrong_kernels(w, D, T):
    B = 10
    x, ga, be, proj = _pool_inputs(B, max(T, 2), w, D, seed=w + D)
    z = x[:, 0]
    for out_f16 in (False, True):
        for normalize in (False, True):
            f, e_f, ref, bound = R.pool_ln_proj_bound(z, ga, be, proj, out_f16, normalize)
            store = (lambda t: t.half()) if out_f16 else (lambda t: t.float())  # noqa: E731
            what = "w=%d D=%d f16=%d normalize=%d" % (w, D, out_f16, normalize)
            assert R.within(store(ref), ref, bound), what
            # the right operation in fp32: LN in fp32, the projection in fp32, normalised in fp32
            zf = _ln_fp32_unrounded(z, ga, be)
            ff = zf @ proj.float()
            assert R.within(ff, f, e_f), what
            assert R.within(store(ff / ff.norm(dim=-1, keepdim=True) if normalize else ff), ref, bound), what

            def out_of(fv):
                return store(fv / fv.norm(dim=-1, keepdim=True) if normalize else fv)

            dropped = f.clone()
            dropped[:, -1] = 0
            variants = {
                "the last output column dropped": out_of(dropped),
                "token 1 pooled instead of token 0": R.pool_ln_proj_bound(x[:, 1], ga, be, proj, out_f16, normalize)[2],
                "an LN without gamma": R.pool_ln_proj_bound(z, ga, be, proj, out_f16, normalize, gamma_off=True)[2],
            }
            for name, y in variants.items():
                assert not R.within(store(y), ref, bound), "%s: the bound accepts %s" % (what, name)


def _ln_fp32_unrounded(z, ga, be):
    zf = z.float()
    mu = zf.mean(-1, keepdim=True)
    d = zf - mu
    return d * torch.rsqrt((d * d).mean(-1, keepdim=True) + 1e-5) * ga + be


@pytest.mark.parametrize("w,D", R.mean_proj_cases())
def test_masked_mean_bound_rejects_wrong_lengths(w, D):
    B, T = 12, 9
    g = torch.Generator().manual_seed(w * 3 + D)
    x = torch.randn(B, T, w, generator=g).bfloat16()
    lengths = torch.arange(B) % (T - 2) + 2                      # 2 .. T - 1: len - 1 and len + 1 are both rows
    projT = torch.randn(w, D, generator=g) * w ** -0.5
    for bias in (None, torch.randn(D, generator=g) * 0.1):
        for out_f16 in (False, True):
            for normalize in (False, True):
                store = (lambda t: t.half()) if out_f16 else (lambda t: t.float())  # noqa: E731
                f, e_f, ref, bound = R.masked_mean_proj_bound(x, lengths, projT, bias, out_f16, normalize)
                what = "w=%d D=%d bias=%d f16=%d normalize=%d" % (w, D, bias is not None, out_f16, normalize)
                assert R.within(store(ref), ref, bound), what
                live = (torch.arange(T)[None, :] < lengths[:, None])[:, :, None]
                mf = (x.float() * live).sum(1) / lengths[:, None].float()
                ff = mf @ projT + (0 if bias is None else bias)
                assert R.within(ff, f, e_f), what
                for k in (1, -1):
                    y = R.masked_mean_proj_bound(x, lengths, projT, bias, out_f16, normalize, length_offset=k)[2]
                    assert not R.within(store(y), ref, bound), "%s: the bound accepts a mean over len %+d rows" % (
                        what, k)


def test_every_table_entry_maps_to_a_case():
    """Each CLIP of model.ARCHS and xlmr_clip.XLMR_CLIP_ARCHS, and each encoder of mclip.MCLIP_ARCHS and the XLM-R
    CLIPs, reaches the kernel cases of test_embed_kernels_gpu.py at its own shapes."""
    from clip_retrieval_b200 import mclip

    ln = {w for w, _ in R.layernorm_cases()}
    ln_rows = {(w, r) for w, r in R.layernorm_cases()}
    im2col = {(S, p) for S, p, _ in R.im2col_cases()}
    text = {w for w, _, _ in R.text_embed_cases()}
    pool = {(w, D, T) for w, D, T in R.pool_cases()}
    mean = set(R.mean_proj_cases())
    assert set(R.LN_TEMPLATE_WIDTHS) <= ln
    assert {math.ceil(w / 256) for w in R.LN_TEMPLATE_WIDTHS} == set(range(1, 9))
    for name, a in R.clip_archs().items():
        T = R.vision_tokens(a)
        assert a.vision.width in ln and any(w == a.vision.width and r > R.LN_PERSISTENT_ROWS for w, r in ln_rows), name
        assert (a.image_size, a.patch) in im2col, name
        assert (a.vision.width, a.embed_dim, T) in pool, name
        if a.text.width:
            assert a.text.width in ln and a.text.width in text, name
            assert (a.text.width, a.embed_dim, a.context_length) in pool, name
    for name, e in R.encoder_archs().items():
        assert e.width in ln and e.layer_norm_eps in R.LN_EPS, name
    for name, e in mclip.MCLIP_ARCHS.items():
        assert (e.width, e.out_dim) in mean, name
    assert any(D % 64 for _, D, _ in pool) and any(w == 200 for w, _, _ in pool)
