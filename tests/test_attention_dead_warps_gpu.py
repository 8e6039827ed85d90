"""Head-dim-64 attention with key lengths at every position of the last query tile.  A warp whose 16 query rows all
lie at or past len[b] skips its softmax and stores, and those rows are zeroed with the tail past the last tile: every
len in 1..T of one batch (so every count of such warps, and every 16-row boundary) gives the float64 attention of the
sample's own tokens on rows < len and exact zeros on the rest.  The output starts as NaN, so a row nobody writes
fails."""
import pytest

from test_embed_gpu import assert_attention_close, attention_ref64
from test_mclip_gpu import run_attention_len

pytestmark = pytest.mark.gpu


@pytest.mark.timeout(300)
@pytest.mark.parametrize("T", [77, 257, 320])
def test_every_key_length_of_one_batch(T):
    import torch

    heads, hd = 2, 64
    w = heads * hd
    lengths = list(range(1, T + 1))
    B = len(lengths)
    g = torch.Generator(device="cuda").manual_seed(31 * T)
    qkv = torch.randn(B * T, 3 * w, device="cuda", generator=g).bfloat16()
    out = run_attention_len(qkv, lengths, B, T, heads, w).view(B, T, w)
    for b, L in enumerate(lengths):
        src = qkv.view(B, T, 3 * w)[b, :L].contiguous()
        ref, bound, _ = attention_ref64(src, 1, L, heads, hd, 0)
        assert_attention_close(out[b, :L], ref, bound, "T=%d len=%d" % (T, L))
        assert bool((out[b, L:] == 0).all()), "T=%d len=%d: rows past the length are not zero" % (T, L)
