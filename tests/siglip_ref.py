"""fp32 forward of open_clip's SigLIP towers from a state_dict in open_clip's key layout (visual.trunk.* as timm names
it, text.*), written from the model's definition rather than from the library's kernels:

  image: x = patch_embed(px) + pos_embed; x = blocks(x); x = norm(x);
         attn_pool: q = q(latent), k | v = kv(x), o = proj(SDPA(q, k, v)), o = o + mlp(norm(o)); features = o[:, 0]
  text:  x = token_embedding[ids] + positional_embedding; x = resblocks(x) (no mask); features =
         text_projection(ln_final(x)[:, -1])

Pre-LN blocks, erf GELU, LayerNorm eps 1e-6.  `tests/golden/make_siglip_golden.py` pins this against transformers'
SiglipModel on a tiny config."""
import numpy as np

EPS = 1e-6


def _t(x):
    import torch

    return x if isinstance(x, torch.Tensor) else torch.as_tensor(np.asarray(x))


def _sd32(sd):
    return {k: _t(v).float() for k, v in sd.items()}


def _ln(x, sd, name):
    import torch.nn.functional as F

    return F.layer_norm(x, x.shape[-1:], sd[name + ".weight"], sd[name + ".bias"], EPS)


def _lin(x, sd, name):
    return x @ sd[name + ".weight"].t() + sd[name + ".bias"]


def _mha(q, k, v, heads, causal=False):
    """q [B, Tq, w], k / v [B, T, w] -> [B, Tq, w]; softmax(q k^T hd^-0.5) v per head, no mask (unless causal)."""
    import torch

    B, Tq, w = q.shape
    T, hd = k.shape[1], w // heads
    q = q.view(B, Tq, heads, hd).transpose(1, 2)
    k = k.view(B, T, heads, hd).transpose(1, 2)
    v = v.view(B, T, heads, hd).transpose(1, 2)
    s = (q @ k.transpose(-1, -2)) * hd ** -0.5
    if causal:
        s = s.masked_fill(torch.ones(Tq, T, dtype=torch.bool).triu_(1), float("-inf"))
    p = torch.softmax(s, -1)
    return (p @ v).transpose(1, 2).reshape(B, Tq, w)


def _gelu(x):
    import torch.nn.functional as F

    return F.gelu(x)


def image_features(sd, arch, px, wrong=()):
    """px fp32 [B, 3, S, S] -> raw image features [B, D] (torch fp32).  `wrong` names deliberate errors, for the tests
    that show the tower bar can fail: "pool_no_residual" (the head's MLP residual dropped), "kv_before_norm" (K / V
    from the trunk before its final norm)."""
    import torch.nn.functional as F

    sd = _sd32(sd)
    v, p = arch.vision, arch.patch
    tr = "visual.trunk."
    x = F.conv2d(_t(px).float(), sd[tr + "patch_embed.proj.weight"], sd[tr + "patch_embed.proj.bias"], stride=p)
    x = x.flatten(2).transpose(1, 2) + sd[tr + "pos_embed"]
    for i in range(v.layers):
        b = "%sblocks.%d." % (tr, i)
        h = _ln(x, sd, b + "norm1")
        q, k, vv = _lin(h, sd, b + "attn.qkv").chunk(3, -1)
        x = x + _lin(_mha(q, k, vv, v.heads), sd, b + "attn.proj")
        x = x + _lin(_gelu(_lin(_ln(x, sd, b + "norm2"), sd, b + "mlp.fc1")), sd, b + "mlp.fc2")
    if "kv_before_norm" not in wrong:
        x = _ln(x, sd, tr + "norm")
    a = tr + "attn_pool."
    B = x.shape[0]
    q = _lin(sd[a + "latent"].expand(B, -1, -1), sd, a + "q")
    k, vv = _lin(x, sd, a + "kv").chunk(2, -1)
    o = _lin(_mha(q, k, vv, v.heads), sd, a + "proj")
    m = _lin(_gelu(_lin(_ln(o, sd, a + "norm"), sd, a + "mlp.fc1")), sd, a + "mlp.fc2")
    o = m if "pool_no_residual" in wrong else o + m
    return o[:, 0]


def text_features(sd, arch, ids, wrong=()):
    """ids int [B, context_length] -> raw text features [B, D] (torch fp32).  `wrong`: "causal" (CLIP's causal mask),
    "eot_pool" (pooled at the first largest id, CLIP's rule, instead of the last position)."""
    sd = _sd32(sd)
    t = arch.text
    ids = _t(ids).long()
    x = sd["text.token_embedding.weight"][ids] + sd["text.positional_embedding"][: ids.shape[1]]
    for i in range(t.layers):
        b = "text.transformer.resblocks.%d." % i
        h = _ln(x, sd, b + "ln_1")
        q, k, v = (h @ sd[b + "attn.in_proj_weight"].t() + sd[b + "attn.in_proj_bias"]).chunk(3, -1)
        x = x + _lin(_mha(q, k, v, t.heads, "causal" in wrong), sd, b + "attn.out_proj")
        x = x + _lin(_gelu(_lin(_ln(x, sd, b + "ln_2"), sd, b + "mlp.c_fc")), sd, b + "mlp.c_proj")
    x = _ln(x, sd, "text.ln_final")
    if "eot_pool" in wrong:
        import torch

        return _lin(x[torch.arange(x.shape[0]), ids.argmax(-1)], sd, "text.text_projection")
    return _lin(x[:, -1], sd, "text.text_projection")
