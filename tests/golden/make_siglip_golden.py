"""Regenerate tests/golden/siglip_tiny.npz: transformers' SiglipModel (an implementation independent of this
repository) at a tiny seeded config, its weights converted to open_clip's SigLIP key layout, and the raw features it
computes for a few images and captions.  Weights and inputs are regenerated from their seeds (`state_dict()`,
`inputs()`), so only the features are stored.  The conversion (HF names -> visual.trunk.* / text.*) is the recalled part;
the golden pins the arithmetic of tests/siglip_ref.py and of the GPU towers.

Config: width 144 with 2 heads (head dim 72, the HD % 16 == 8 tail), 2 layers and MLP 288 per tower, 32 px images in
8 px patches (16 tokens), text context 16, vocab 300, erf GELU, LayerNorm eps 1e-6.

    python tests/golden/make_siglip_golden.py
"""
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "siglip_tiny.npz")
W, HEADS, LAYERS, MLP, S, P, CTX, VOCAB = 144, 2, 2, 288, 32, 8, 16, 300


def hf_model():
    from transformers import SiglipConfig, SiglipModel

    common = dict(hidden_size=W, intermediate_size=MLP, num_hidden_layers=LAYERS, num_attention_heads=HEADS,
                  hidden_act="gelu", layer_norm_eps=1e-6, attention_dropout=0.0)
    cfg = SiglipConfig(text_config=dict(common, vocab_size=VOCAB, max_position_embeddings=CTX, projection_size=W,
                                        pad_token_id=1, bos_token_id=2, eos_token_id=1),
                       vision_config=dict(common, image_size=S, patch_size=P, num_channels=3))
    torch.manual_seed(0)
    model = SiglipModel(cfg).eval()
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        # non-trivial LayerNorm affines, biases and embeddings (the default init leaves many of them 1 / 0)
        for name, p in model.named_parameters():
            if name.endswith("weight") and p.dim() == 1:
                p.copy_(1.0 + 0.1 * torch.randn(p.shape, generator=g))
            elif name.endswith("bias") or name.endswith("probe"):
                p.copy_(0.05 * torch.randn(p.shape, generator=g))
            elif "embedding" in name:
                p.copy_((W ** -0.5) * torch.randn(p.shape, generator=g))
            else:
                p.copy_(p.shape[-1] ** -0.5 * torch.randn(p.shape, generator=g))
    model.config._attn_implementation = "eager"
    return model


def to_open_clip(hf):
    """HF SiglipModel parameter names -> open_clip's SigLIP layout."""
    sd = {k: v.detach().clone().float() for k, v in hf.items()}
    out = {}
    v, t = "vision_model.", "text_model."
    out["visual.trunk.patch_embed.proj.weight"] = sd[v + "embeddings.patch_embedding.weight"]
    out["visual.trunk.patch_embed.proj.bias"] = sd[v + "embeddings.patch_embedding.bias"]
    out["visual.trunk.pos_embed"] = sd[v + "embeddings.position_embedding.weight"][None]
    for i in range(LAYERS):
        s, d = "%sencoder.layers.%d." % (v, i), "visual.trunk.blocks.%d." % i
        for a, b in (("norm1", "layer_norm1"), ("norm2", "layer_norm2"), ("attn.proj", "self_attn.out_proj"),
                     ("mlp.fc1", "mlp.fc1"), ("mlp.fc2", "mlp.fc2")):
            out[d + a + ".weight"], out[d + a + ".bias"] = sd[s + b + ".weight"], sd[s + b + ".bias"]
        out[d + "attn.qkv.weight"] = torch.cat([sd[s + "self_attn.%s_proj.weight" % n] for n in "qkv"], 0)
        out[d + "attn.qkv.bias"] = torch.cat([sd[s + "self_attn.%s_proj.bias" % n] for n in "qkv"], 0)
    out["visual.trunk.norm.weight"], out["visual.trunk.norm.bias"] = sd[v + "post_layernorm.weight"], sd[v + "post_layernorm.bias"]
    h, a = v + "head.", "visual.trunk.attn_pool."
    out[a + "latent"] = sd[h + "probe"]
    ipw, ipb = sd[h + "attention.in_proj_weight"], sd[h + "attention.in_proj_bias"]
    out[a + "q.weight"], out[a + "q.bias"] = ipw[:W], ipb[:W]
    out[a + "kv.weight"], out[a + "kv.bias"] = ipw[W:], ipb[W:]
    out[a + "proj.weight"], out[a + "proj.bias"] = sd[h + "attention.out_proj.weight"], sd[h + "attention.out_proj.bias"]
    out[a + "norm.weight"], out[a + "norm.bias"] = sd[h + "layernorm.weight"], sd[h + "layernorm.bias"]
    for n in ("fc1", "fc2"):
        out[a + "mlp.%s.weight" % n], out[a + "mlp.%s.bias" % n] = sd[h + "mlp.%s.weight" % n], sd[h + "mlp.%s.bias" % n]
    out["text.token_embedding.weight"] = sd[t + "embeddings.token_embedding.weight"]
    out["text.positional_embedding"] = sd[t + "embeddings.position_embedding.weight"]
    for i in range(LAYERS):
        s, d = "%sencoder.layers.%d." % (t, i), "text.transformer.resblocks.%d." % i
        for a_, b in (("ln_1", "layer_norm1"), ("ln_2", "layer_norm2"), ("attn.out_proj", "self_attn.out_proj"),
                      ("mlp.c_fc", "mlp.fc1"), ("mlp.c_proj", "mlp.fc2")):
            out[d + a_ + ".weight"], out[d + a_ + ".bias"] = sd[s + b + ".weight"], sd[s + b + ".bias"]
        out[d + "attn.in_proj_weight"] = torch.cat([sd[s + "self_attn.%s_proj.weight" % n] for n in "qkv"], 0)
        out[d + "attn.in_proj_bias"] = torch.cat([sd[s + "self_attn.%s_proj.bias" % n] for n in "qkv"], 0)
    out["text.ln_final.weight"], out["text.ln_final.bias"] = sd[t + "final_layer_norm.weight"], sd[t + "final_layer_norm.bias"]
    out["text.text_projection.weight"], out["text.text_projection.bias"] = sd[t + "head.weight"], sd[t + "head.bias"]
    return out


def state_dict():
    """The golden's weights in open_clip's layout."""
    return to_open_clip(hf_model().state_dict())


def inputs():
    g = torch.Generator().manual_seed(2)
    px = torch.randn(4, 3, S, S, generator=g)
    ids = torch.randint(3, VOCAB, (4, CTX), generator=g)
    ids[0, 5:] = 1      # a short caption: </s> then pads (pad id 1)
    ids[1, 11:] = 1
    return px, ids


def main():
    model = hf_model()
    px, ids = inputs()
    with torch.no_grad():
        img = model.vision_model(pixel_values=px).pooler_output
        txt = model.text_model(input_ids=ids).pooler_output
    np.savez_compressed(OUT, image=img.numpy(), text=txt.numpy(), source="transformers SiglipModel fp32")
    print("wrote", OUT, img.shape, txt.shape)


if __name__ == "__main__":
    main()
