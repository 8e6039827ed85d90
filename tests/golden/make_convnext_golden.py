"""Generate tests/golden/clip_tiny-convnext.npz: the image features of a tiny ConvNeXt CLIP computed with
`transformers.ConvNextModel` (an independent implementation of the trunk) and open_clip's head applied to its pooler
output, written independently of oracle/convnext_ref.py.  Weights: model.synthetic_state_dict(TINY, 0), mapped from
open_clip's layout to HuggingFace's.  Run from the repo root:
    python tests/golden/make_convnext_golden.py
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import clip_retrieval_b200 as m  # noqa: E402
from oracle import clip_ref  # noqa: E402

# widths 64..256 (the kernels' multiples of 64), depths 1, 1, 2, 1, 64 px (maps 16, 8, 4, 2), the MLP head
TINY = m.ConvNeXtArch(64, 64, (1, 1, 2, 1), (64, 128, 192, 256), True, m.Tower(128, 2, 2, 512))
N = 5
OUT = os.path.join(ROOT, "tests", "golden", "clip_tiny-convnext.npz")


def hf_state_dict(sd, arch):
    """open_clip's visual.trunk.* -> transformers.ConvNextModel's keys."""
    t, out = "visual.trunk.", {}
    out["embeddings.patch_embeddings.weight"] = sd[t + "stem.0.weight"]
    out["embeddings.patch_embeddings.bias"] = sd[t + "stem.0.bias"]
    out["embeddings.layernorm.weight"] = sd[t + "stem.1.weight"]
    out["embeddings.layernorm.bias"] = sd[t + "stem.1.bias"]
    for s, n in enumerate(arch.depths):
        p, q = "%sstages.%d." % (t, s), "encoder.stages.%d." % s
        if s > 0:
            for i in (0, 1):
                for a in ("weight", "bias"):
                    out[q + "downsampling_layer.%d.%s" % (i, a)] = sd[p + "downsample.%d.%s" % (i, a)]
        for j in range(n):
            b, c = "%sblocks.%d." % (p, j), "%slayers.%d." % (q, j)
            out[c + "layer_scale_parameter"] = sd[b + "gamma"]
            for src, dst in (("conv_dw", "dwconv"), ("norm", "layernorm"), ("mlp.fc1", "pwconv1"), ("mlp.fc2", "pwconv2")):
                for a in ("weight", "bias"):
                    out[c + dst + "." + a] = sd[b + src + "." + a]
    out["layernorm.weight"] = sd[t + "head.norm.weight"]
    out["layernorm.bias"] = sd[t + "head.norm.bias"]
    return out


@torch.no_grad()
def main():
    from transformers import ConvNextConfig, ConvNextModel

    sd = m.synthetic_state_dict(TINY, seed=0)
    # HF hard-codes eps 1e-6 in the stem, block and downsample LayerNorms; its final one reads layer_norm_eps
    cfg = ConvNextConfig(num_channels=3, patch_size=4, num_stages=4, hidden_sizes=list(TINY.dims),
                         depths=list(TINY.depths), hidden_act="gelu", layer_norm_eps=1e-6, layer_scale_init_value=1e-6,
                         drop_path_rate=0.0, image_size=TINY.image_size)
    model = ConvNextModel(cfg).eval()
    missing, unexpected = model.load_state_dict(hf_state_dict(sd, TINY), strict=True)
    assert not missing and not unexpected
    px = clip_ref.synth_images(N, TINY)
    pooled = model(pixel_values=px).pooler_output
    h = F.gelu(pooled @ sd["visual.head.mlp.fc1.weight"].t() + sd["visual.head.mlp.fc1.bias"])
    feat = h @ sd["visual.head.mlp.fc2.weight"].t()
    np.savez(OUT, image=feat.numpy().astype(np.float32))
    print("wrote", OUT, feat.shape)


if __name__ == "__main__":
    main()
