"""Attention past the whole-K/V kernel's shared-memory limit: the streaming kernel (K and V through a ring of 64-key
stages) against the float64 reference, on both sides of the switch for every head dim, at long sequences, with
per-sample key lengths, with one-hot V probes on the stage boundaries, and batch by batch against single samples."""
import pytest

from test_embed_gpu import assert_attention_close, attention_ref64, run_attention
from test_mclip_gpu import run_attention_len

pytestmark = pytest.mark.gpu

# the longest T the whole-K/V kernel takes per head dim: 2 * ceil32(T) * (hd + 8) * 2 bytes <= 200 KB
LONGEST_WHOLE = {64: 704, 80: 576, 96: 480, 128: 352}
STAGE = 64


def _qkv(B, T, w, seed):
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(B * T, 3 * w, device="cuda", generator=g).bfloat16()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("causal", [0, 1])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("hd", [64, 80, 96, 128])
def test_both_sides_of_the_switch(hd, B, causal):
    """The longest T the whole-K/V kernel takes, T + 1 (the first streamed shape) and T + 1 + one ring stage."""
    heads = 2
    w = heads * hd
    top = LONGEST_WHOLE[hd]
    for T in (top, top + 1, top + 1 + STAGE):
        qkv = _qkv(B, T, w, 7 * T + hd + causal)
        out = run_attention(qkv, B, T, heads, w, causal)
        ref, bound, _ = attention_ref64(qkv, B, T, heads, hd, causal)
        assert_attention_close(out, ref, bound, "hd=%d B=%d T=%d causal=%d" % (hd, B, T, causal))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("T,heads,hd,causal", [(730, 16, 80, 0), (730, 2, 80, 1), (1025, 2, 64, 1), (1025, 2, 64, 0)])
def test_long_sequences(T, heads, hd, causal):
    B, w = 2, heads * hd
    qkv = _qkv(B, T, w, T + hd + causal)
    out = run_attention(qkv, B, T, heads, w, causal)
    ref, bound, _ = attention_ref64(qkv, B, T, heads, hd, causal)
    assert_attention_close(out, ref, bound, "T=%d hd=%d causal=%d" % (T, hd, causal))


@pytest.mark.timeout(300)
def test_per_sample_lengths():
    """Each sample attends to its own keys only; its rows past the length are exactly zero in a NaN-filled buffer
    (a 128-row chunk wholly past the length loads nothing and writes zeros)."""
    T, heads, hd = 730, 2, 80
    w = heads * hd
    lengths = [1, 2, 127, 128, 129, 729, 730]
    B = len(lengths)
    qkv = _qkv(B, T, w, 4242)
    out = run_attention_len(qkv, lengths, B, T, heads, w).view(B, T, w)
    for b, L in enumerate(lengths):
        src = qkv.view(B, T, 3 * w)[b, :L].contiguous()
        ref, bound, _ = attention_ref64(src, 1, L, heads, hd, 0)
        assert_attention_close(out[b, :L], ref, bound, "len=%d" % L)
        assert bool((out[b, L:] == 0).all()), "len=%d: rows past the length are not zero" % L


@pytest.mark.timeout(300)
@pytest.mark.parametrize("causal", [0, 1])
@pytest.mark.parametrize("T,hd", [(730, 80), (705, 64), (481, 96), (353, 128)])
def test_one_hot_v_probes_on_stage_boundaries(T, hd, causal):
    """V is zero except one 1.0 per (sample, head) at key t, dim j: that output dim is P[r, t] alone and every other
    output is exactly 0.  Keys 0, 63, 64, 65 and T - 1 sit on the ring's stage boundaries; 5 samples per head with
    different dims catch a stage read out of order or a key of the neighbouring sample."""
    import torch

    keys = [0, 63, 64, 65, T - 1]
    dims = [0, 7, 8, 33, hd - 1]
    B, heads = 5, len(keys)
    w = heads * hd
    g = torch.Generator(device="cuda").manual_seed(T + hd + causal)
    qkv = torch.randn(B * T, 3 * w, device="cuda", generator=g)
    view = qkv.view(B, T, 3, heads, hd)
    view[:, :, 2] = 0.0
    probe = {}
    for h, t in enumerate(keys):
        for b in range(B):
            j = dims[(b + h) % len(dims)]
            view[b, t, 2, h, j] = 1.0
            probe[(b, h)] = (t, j)
    qkv = qkv.bfloat16()
    out = run_attention(qkv, B, T, heads, w, causal).view(B, T, heads, hd).double()
    _, _, P = attention_ref64(qkv, B, T, heads, hd, causal)
    want = torch.zeros(B, T, heads, hd, dtype=torch.float64, device="cuda")
    for (b, h), (t, j) in probe.items():
        want[b, :, h, j] = P[b, h, :, t]
    zero = want == 0
    assert bool((out[zero] == 0).all()), "%d outputs that must be exactly 0 are not (first: %s)" % (
        int((out[zero] != 0).sum()), torch.nonzero(zero & (out != 0))[:1].tolist())
    err = (out[~zero] - want[~zero]).abs()
    assert bool((err <= (2.0 ** -7 + 2.0 ** -12) * want[~zero]).all()), \
        "probe P[r, t]: max rel err %g" % (err / want[~zero]).max().item()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("causal", [0, 1])
def test_batch_independence(causal):
    """Sample b of a batch equals the same sample run alone, bit for bit."""
    import torch

    B, T, heads, hd = 4, 730, 3, 80
    w = heads * hd
    qkv = _qkv(B, T, w, 99 + causal)
    full = run_attention(qkv, B, T, heads, w, causal).view(B, T, w)
    for b in range(B):
        one = run_attention(qkv.view(B, T, 3 * w)[b].contiguous(), 1, T, heads, w, causal)
        assert torch.equal(full[b], one), b
