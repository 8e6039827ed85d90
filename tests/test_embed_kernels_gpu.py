"""Kernel-level parity of the embed path's non-GEMM kernels against float64 on their own inputs: LayerNorm (both
epsilon entries, every template width, the persistent grid's edges, serving batches, in place), the vision tower's
front (im2col + class rows), the text tower's front (token + positional embedding, the EOT index), the pooled
LN -> projection -> normalise end of both towers, and the M-CLIP masked-mean head.  Shapes come from the model tables
(embed_kernels_ref.py); the bounds and their derivations are there too, and test_embed_kernels_cpu.py shows that
each bound rejects named wrong kernels.  Rows a kernel must not read are NaN, and outputs start as NaN, so a wrong
read or a missing write cannot hide inside a tolerance."""
import math

import numpy as np
import pytest

import embed_kernels_ref as R

pytestmark = pytest.mark.gpu
NAN = float("nan")


def _stream():
    import torch

    return torch.cuda.current_stream().cuda_stream


# ---- LayerNorm ------------------------------------------------------------------------------------------------------

def _layernorm(x, out, ga, be, eps):
    """eps None: the fixed-epsilon entry (1e-5); else the entry with the epsilon as an argument."""
    from clip_retrieval_b200._lib import lib, check

    rows, w = x.shape
    if eps is None:
        check(lib.b200_layernorm_bf16_device(x.data_ptr(), out.data_ptr(), ga.data_ptr(), be.data_ptr(), rows, w, 0,
                                             _stream()), "layernorm")
    else:
        check(lib.b200_layernorm_eps_bf16_device(x.data_ptr(), out.data_ptr(), ga.data_ptr(), be.data_ptr(), rows, w,
                                                 eps, 0, _stream()), "layernorm_eps")


def check_layernorm(w, rows, runs):
    """Each (eps, entry) of `runs` (entry None: the fixed-epsilon entry, else the epsilon passed) against
    R.layernorm_bound (see its docstring for the derivation) on rows of every class of R.layernorm_inputs; constant
    rows give bf16(beta) exactly; the in-place call (in == out) stores the same bits as the out-of-place one.
    -> {(eps, entry): output}."""
    import torch

    x, ga, be, cls = R.layernorm_inputs(rows, w, seed=rows * 31 + w, device="cuda")
    const = cls == 4
    outs = {}
    for eps, entry in runs:
        out = torch.full_like(x, NAN)
        _layernorm(x, out, ga, be, entry)
        ref, bound = R.layernorm_bound(x, ga, be, eps, "rows")
        what = "w=%d rows=%d eps=%g %s entry" % (w, rows, eps, "fixed" if entry is None else "eps")
        R.assert_within(out[~const], ref[~const], bound[~const], what)
        assert torch.equal(out[const], be.bfloat16().expand(int(const.sum()), w)), what + ": constant rows"
        inplace = x.clone()
        _layernorm(inplace, inplace, ga, be, entry)
        assert torch.equal(inplace, out), what + ": in place differs"
        outs[(eps, entry)] = out
    return outs


@pytest.mark.timeout(300)
@pytest.mark.parametrize("w,rows", R.layernorm_cases())
def test_layernorm_matches_float64(w, rows):
    """Both entries through check_layernorm, at eps 1e-5 and 1e-12; the fixed entry stores the same bits as the eps
    entry at 1e-5."""
    import torch

    outs = check_layernorm(w, rows, ((1e-5, None), (1e-5, 1e-5), (1e-12, 1e-12)))
    assert torch.equal(outs[(1e-5, None)], outs[(1e-5, 1e-5)])


# ---- vision front: im2col + class rows ------------------------------------------------------------------------------

@pytest.mark.timeout(120)
@pytest.mark.parametrize("S,p,w", R.im2col_cases())
@pytest.mark.parametrize("B", [1, 3])
def test_im2col_and_class_rows_bit_exact(S, p, w, B):
    """Patch rows equal unfold() of the bf16-rounded pixels bit for bit; the pad columns [3 p^2, Kp) and the rows past
    B g^2 keep their NaN (the model zeroes the pad once and relies on nobody writing it); row b T of x is bf16(cls)
    and every other row of x is untouched."""
    import torch
    from clip_retrieval_b200._lib import lib, check

    g = S // p
    k = 3 * p * p
    Kp = (k + 63) // 64 * 64
    T = g * g + 1
    gen = torch.Generator(device="cuda").manual_seed(S * 7 + p + B)
    px = torch.randn(B, 3, S, S, device="cuda", generator=gen) * 2
    cls = torch.randn(w, device="cuda", generator=gen)
    cols = torch.full((B * g * g + 2, Kp), NAN, device="cuda", dtype=torch.bfloat16)
    x = torch.full((B * T + 1, w), NAN, device="cuda", dtype=torch.bfloat16)
    check(lib.b200_vision_front_bf16_device(px.data_ptr(), B, S, p, Kp, cols.data_ptr(), cls.data_ptr(), T, w,
                                            x.data_ptr(), 0, _stream()), "vision_front")
    torch.cuda.synchronize()
    ref = torch.nn.functional.unfold(px.bfloat16().float(), kernel_size=p, stride=p)      # [B, 3 p p, g g]
    ref = ref.transpose(1, 2).reshape(B * g * g, k).bfloat16()
    assert torch.equal(cols[:B * g * g, :k], ref), "patch values"
    assert bool(cols[:, k:].isnan().all()), "a pad column was written"
    assert bool(cols[B * g * g:].isnan().all()), "a row past B g^2 was written"
    xv = x[:B * T].view(B, T, w)
    assert torch.equal(xv[:, 0], cls.bfloat16().expand(B, w)), "class rows"
    assert bool(xv[:, 1:].isnan().all()) and bool(x[B * T:].isnan().all()), "a row other than a class row was written"


# ---- text front: token + positional embedding, EOT index ------------------------------------------------------------

@pytest.mark.timeout(120)
@pytest.mark.parametrize("w,T,vocab", R.text_embed_cases())
def test_text_embed_bit_exact(w, T, vocab):
    """x[b T + t] = bf16(float(tok_emb[clamp(tok, 0, vocab - 1)]) + pos[t]) bit for bit, at B = 3 (t = row mod T),
    with ids -1, 0, vocab - 1, vocab and vocab + 100 among the tokens; the row past B T is not written."""
    import torch
    from clip_retrieval_b200._lib import lib, check

    B = 3
    gen = torch.Generator(device="cuda").manual_seed(w + T)
    tok_emb = torch.randn(vocab, w, device="cuda", generator=gen).bfloat16()
    pos = torch.randn(T, w, device="cuda", generator=gen) * 0.1
    tokens = torch.randint(0, vocab, (B, T), device="cuda", generator=gen)
    edges = torch.tensor([-1, 0, vocab - 1, vocab, vocab + 100], device="cuda")
    tokens[0, :5] = edges
    tokens[1, T - 5:] = edges
    tokens[2, T // 2:T // 2 + 5] = edges.flip(0)
    x = torch.full((B * T + 1, w), NAN, device="cuda", dtype=torch.bfloat16)
    check(lib.b200_text_embed_bf16_device(tokens.data_ptr(), tok_emb.data_ptr(), pos.data_ptr(), x.data_ptr(), B, T, w,
                                          vocab, 0, _stream()), "text_embed")
    torch.cuda.synchronize()
    ref = (tok_emb[tokens.clamp(0, vocab - 1)].float() + pos[None]).bfloat16().view(B * T, w)
    assert torch.equal(x[:B * T], ref)
    assert bool(x[B * T:].isnan().all())


@pytest.mark.timeout(120)
@pytest.mark.parametrize("B", [1, 127, 128, 129, 1024])
def test_token_argmax_first_maximum(B):
    """The EOT index is the first maximum of each row, exactly: rows of SOT, words, EOT and padding; EOT at t = 0 and
    at t = T - 1; two equal maxima; an all-zero row (index 0)."""
    import torch
    from clip_retrieval_b200._lib import lib, check

    T, vocab = 77, 49408
    rng = np.random.default_rng(B)
    tok = np.zeros((B, T), dtype=np.int64)
    for b in range(B):
        kind = b % 5
        if kind == 0:
            n = int(rng.integers(0, T - 1))
            tok[b, 0], tok[b, 1:n + 1], tok[b, n + 1] = vocab - 2, rng.integers(1, vocab - 2, n), vocab - 1
        elif kind in (1, 2):
            tok[b] = rng.integers(0, vocab - 1, T)
            tok[b, T - 1 if kind == 1 else 0] = vocab - 1
        elif kind == 3:
            tok[b] = rng.integers(0, 1000, T)
            i, j = sorted(rng.choice(T, 2, replace=False))
            tok[b, i] = tok[b, j] = 5000
    want = tok.argmax(1)
    d_tok = torch.as_tensor(tok, device="cuda")
    idx = torch.full((B + 1,), -7, dtype=torch.int32, device="cuda")
    check(lib.b200_token_argmax_device(d_tok.data_ptr(), B, T, idx.data_ptr(), 0, _stream()), "token_argmax")
    got = idx.cpu().numpy()
    assert np.array_equal(got[:B], want) and got[B] == -7
    if B >= 5:
        assert set(want[1:5]) >= {T - 1, 0}


# ---- tower end: pooled LN -> projection -> normalise ------------------------------------------------------------------

def _pool_run(x, B, T, pool_idx, ga, be, proj, out_f16, normalize):
    import torch
    from clip_retrieval_b200._lib import lib, check

    w, D = proj.shape
    feat = torch.full((B, D), NAN, device="cuda")
    out = torch.full((B, D), NAN, device="cuda", dtype=torch.float16 if out_f16 else torch.float32)
    check(lib.b200_pool_ln_proj_device(x.data_ptr(), B, T, w, 0 if pool_idx is None else pool_idx.data_ptr(),
                                       ga.data_ptr(), be.data_ptr(), proj.data_ptr(), D, feat.data_ptr(),
                                       out.data_ptr(), int(out_f16), normalize, 0, _stream()), "pool_ln_proj")
    torch.cuda.synchronize()
    return feat, out


def _eot_rows(B, T):
    """Per-sample EOT rows: T - 1 for sample 0 (its +1 neighbour is the NaN guard row when B = 1), 0 for sample 1,
    then spread over 0 .. T - 1; the last sample's is T - 1 too."""
    t = [(b * 37 + T - 1) % T for b in range(B)]
    if B > 1:
        t[1], t[-1] = 0, T - 1
    return t


@pytest.mark.timeout(300)
@pytest.mark.parametrize("w,D,T", R.pool_cases())
@pytest.mark.parametrize("B", [1, 3, 1024])
def test_pool_ln_proj_matches_float64(w, D, T, B):
    """Raw features and stored rows against R.pool_ln_proj_bound, pooling token 0 (no index) and per-sample EOT rows
    (an index), fp16 and fp32 out, normalised or not.  Every row but the pooled ones is NaN, and so is a guard row
    past the last sample: a read of any other row poisons the output."""
    import torch

    gen = torch.Generator(device="cuda").manual_seed(w * 3 + D + B)
    z, ga, be, _ = R.layernorm_inputs(B, w, seed=w + D + B, device="cuda")
    proj = (torch.randn(w, D, device="cuda", generator=gen) * w ** -0.5).bfloat16()
    eot = _eot_rows(B, T)
    for pooled in ([0] * B, eot):
        x = torch.full((B * T + 1, w), NAN, device="cuda", dtype=torch.bfloat16)
        rows = torch.tensor([b * T + t for b, t in enumerate(pooled)], device="cuda")
        x[rows] = z
        idx = None if pooled is not eot else torch.tensor(eot, dtype=torch.int32, device="cuda")
        for out_f16 in (False, True):
            for normalize in (0, 1):
                what = "w=%d D=%d T=%d B=%d %s f16=%d normalize=%d" % (w, D, T, B, "eot" if idx is not None else
                                                                        "token 0", out_f16, normalize)
                feat, out = _pool_run(x, B, T, idx, ga, be, proj, out_f16, normalize)
                f, e_f, ref, bound = R.pool_ln_proj_bound(z, ga, be, proj, out_f16, normalize)
                R.assert_within(feat, f, e_f, what + " feat")
                R.assert_within(out, ref, bound, what)


@pytest.mark.timeout(120)
@pytest.mark.parametrize("w,D,T", [R.pool_cases()[0], R.POOL_EXTRA[0]])
def test_pool_ln_proj_zero_projection_gives_nan_rows(w, D, T):
    """`features /= features.norm()` has no epsilon: a zero projection gives NaN rows when normalised, zeros when not."""
    import torch

    B = 3
    z, ga, be, _ = R.layernorm_inputs(B * T, w, seed=5, device="cuda")
    proj = torch.zeros(w, D, device="cuda", dtype=torch.bfloat16)
    for out_f16 in (False, True):
        feat, out = _pool_run(z, B, T, None, ga, be, proj, out_f16, 1)
        assert bool((feat == 0).all()) and bool(out.isnan().all()), out_f16
        _, out = _pool_run(z, B, T, None, ga, be, proj, out_f16, 0)
        assert bool((out == 0).all()), out_f16


# ---- M-CLIP head: masked mean -> projection (+ bias) -> normalized() -------------------------------------------------

def _mean_proj_run(x, lengths, projT, bias, B, T, out_f16, normalize):
    import torch
    from clip_retrieval_b200._lib import lib, check

    w, D = projT.shape
    d_len = torch.as_tensor(lengths, dtype=torch.int32, device="cuda")
    feat = torch.full((B, D), NAN, device="cuda")
    out = torch.full((B, D), NAN, device="cuda", dtype=torch.float16 if out_f16 else torch.float32)
    check(lib.b200_mean_proj_head_device(x.data_ptr(), B, T, w, d_len.data_ptr(), projT.data_ptr(),
                                         0 if bias is None else bias.data_ptr(), D, feat.data_ptr(), out.data_ptr(),
                                         int(out_f16), normalize, 0, _stream()), "mean_proj_head")
    torch.cuda.synchronize()
    return feat, out


@pytest.mark.timeout(300)
@pytest.mark.parametrize("w,D", R.mean_proj_cases())
@pytest.mark.parametrize("B", [1, 3, 1024])
def test_masked_mean_proj_matches_float64(w, D, B):
    """Raw features and stored rows against R.masked_mean_proj_bound, with and without the bias, fp16 and fp32 out,
    normalised or not.  Rows t >= clamp(len, 1, T) are NaN, as is a guard row past the last sample; lengths include
    0 (read as 1), 1, T and T + 5 (read as T)."""
    import torch

    T = 20
    gen = torch.Generator(device="cuda").manual_seed(w + D * 5 + B)
    lengths = [(0, 1, T, T + 5)[b] if b < 4 else (b * 7) % T + 1 for b in range(B)]
    live = [min(max(n, 1), T) for n in lengths]
    x = torch.full((B * T + 1, w), NAN, device="cuda", dtype=torch.bfloat16)
    vals = torch.randn(B, T, w, device="cuda", generator=gen).bfloat16()
    xv = x[:B * T].view(B, T, w)
    for b, n in enumerate(live):
        xv[b, :n] = vals[b, :n]
    projT = torch.randn(w, D, device="cuda", generator=gen) * w ** -0.5
    bias = torch.randn(D, device="cuda", generator=gen) * 0.1
    d_len = torch.as_tensor(lengths, device="cuda")
    for bb in (None, bias):
        for out_f16 in (False, True):
            for normalize in (0, 1):
                what = "w=%d D=%d B=%d bias=%d f16=%d normalize=%d" % (w, D, B, bb is not None, out_f16, normalize)
                feat, out = _mean_proj_run(x, lengths, projT, bb, B, T, out_f16, normalize)
                f, e_f, ref, bound = R.masked_mean_proj_bound(xv, d_len, projT, bb, out_f16, normalize)
                R.assert_within(feat, f, e_f, what + " feat")
                R.assert_within(out, ref, bound, what)


@pytest.mark.timeout(120)
@pytest.mark.parametrize("w,D", [(1024, 768), (768, 512)])
def test_masked_mean_zero_feature_row_stays_zero(w, D):
    """clip_back's normalized() divides a zero row by 1: a zero projection without bias gives exact zeros, no NaN."""
    import torch

    B, T = 3, 7
    x = torch.randn(B * T, w, device="cuda").bfloat16()
    projT = torch.zeros(w, D, device="cuda")
    for out_f16 in (False, True):
        feat, out = _mean_proj_run(x, [T, 1, 3], projT, None, B, T, out_f16, 1)
        assert bool((feat == 0).all()) and bool((out == 0).all()), out_f16
