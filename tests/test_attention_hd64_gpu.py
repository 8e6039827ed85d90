"""The head-dim-64 wgmma attention kernel (csrc/attention_wgmma.cu) over everything its tiling depends on: every T it
takes (every width of the last key block, every count of query tiles and so every use of the two Q slots of each
warpgroup), causal and not, against the float64 reference and bound of test_embed_gpu.py; the benchmark shape, one
sample at a time against the batched launch; one-hot V probes of the transposed-B V operand; and the model path with
fewer samples than the model was built for (its tensor map covers max_batch samples)."""
import numpy as np
import pytest

from oracle import clip_ref
from test_embed_gpu import _model, assert_attention_close, attention_ref64, run_attention
from test_embed_gpu import test_attention_one_hot_v_probes as one_hot_v_probes

pytestmark = pytest.mark.gpu


@pytest.mark.timeout(300)
@pytest.mark.parametrize("causal", [0, 1])
def test_every_sequence_length_matches_float64(causal):
    import torch

    B, heads, hd = 2, 2, 64
    w = heads * hd
    for T in range(1, 321):
        g = torch.Generator(device="cuda").manual_seed(T * 2 + causal)
        qkv = torch.randn(B * T, 3 * w, device="cuda", generator=g).bfloat16()
        out = run_attention(qkv, B, T, heads, w, causal)
        ref, bound, _ = attention_ref64(qkv, B, T, heads, hd, causal)
        assert_attention_close(out, ref, bound, "T=%d causal=%d" % (T, causal))


@pytest.mark.timeout(300)
def test_benchmark_shape_samples_alone_equal_the_batch():
    """ViT-L/14 image attention at batch 1024: samples 0, 1, 511 and 1023 launched alone reproduce their rows of the
    batched result bit for bit, and are within the float64 bound."""
    import torch

    B, T, heads, hd = 1024, 257, 16, 64
    w = heads * hd
    g = torch.Generator(device="cuda").manual_seed(257)
    qkv = torch.randn(B * T, 3 * w, device="cuda", generator=g).bfloat16()
    full = run_attention(qkv, B, T, heads, w, 0)
    for b in (0, 1, 511, 1023):
        src = qkv[b * T:(b + 1) * T].contiguous()
        one = run_attention(src, 1, T, heads, w, 0)
        assert torch.equal(one, full[b * T:(b + 1) * T]), "sample %d differs from its batched result" % b
        ref, bound, _ = attention_ref64(src, 1, T, heads, hd, 0)
        assert_attention_close(one, ref, bound, "sample %d" % b)


@pytest.mark.timeout(120)
@pytest.mark.parametrize("causal", [0, 1])
@pytest.mark.parametrize("T", [17, 77, 197, 257, 320])
def test_one_hot_v_probes(T, causal):
    one_hot_v_probes(T, 64, causal)


@pytest.mark.timeout(300)
def test_model_below_max_batch_matches_full_batch():
    """Both towers of the tiny config run the wgmma kernel (head dim 64, T = 17 image and 77 causal text); 3 samples
    through a model built for 8 match the same samples in a full batch of 8, and the oracle."""
    model, cfg, sd = _model("tiny", 8)
    px, tk = clip_ref.synth_images(8, cfg), clip_ref.synth_tokens(8, cfg)
    ei8, et8 = model.embed_image(px), model.embed_text(tk)
    ei3, et3 = model.embed_image(px[:3]), model.embed_text(tk[:3])
    for a, b in ((ei3, ei8[:3]), (et3, et8[:3])):
        d = float(np.abs(a.astype(np.float32) - b.astype(np.float32)).max())
        assert d <= 2e-3, "3-sample batch vs full batch: max abs diff %g" % d
    assert (1 - clip_ref.cosine(ei3, clip_ref.mapper_image(sd, cfg, px[:3]))).max() <= 1e-3
    assert (1 - clip_ref.cosine(et3, clip_ref.mapper_text(sd, cfg, tk[:3]))).max() <= 1e-3
