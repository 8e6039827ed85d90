"""Generate tests/golden/clip_tiny-rn.npz: the image features of a tiny ResNet CLIP computed with `torch.nn` modules
(nn.Conv2d, nn.BatchNorm2d in eval mode, nn.AvgPool2d, nn.ReLU) and F.multi_head_attention_forward with separate
q / k / v projections, written independently of oracle/resnet_ref.py.  Weights: model.synthetic_state_dict(TINY, 0).
Run from the repo root:
    python tests/golden/make_rn_golden.py
"""
import os
import sys

import numpy as np
import torch
from torch import nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import clip_retrieval_b200 as m  # noqa: E402
from oracle import clip_ref  # noqa: E402

# width 16 (stem channels 8, attention pool 512 = 8 heads of 64), one block per stage, 64 px (final map 2 x 2, T = 5)
TINY = m.ResNetArch(64, 64, (1, 1, 1, 1), 16, m.Tower(128, 2, 2, 512), quick_gelu=True)
N = 5
OUT = os.path.join(ROOT, "tests", "golden", "clip_tiny-rn.npz")


def _conv(sd, name, cin, cout, k, stride=1):
    c = nn.Conv2d(cin, cout, k, stride=stride, padding=k // 2, bias=False)
    c.weight.data.copy_(sd[name + ".weight"])
    return c


def _bn(sd, name, n):
    b = nn.BatchNorm2d(n)
    for a in ("weight", "bias", "running_mean", "running_var"):
        getattr(b, a).data.copy_(sd[name + "." + a])
    return b.eval()


class Bottleneck(nn.Module):
    def __init__(self, sd, p, cin, planes, stride):
        super().__init__()
        self.c1, self.b1 = _conv(sd, p + "conv1", cin, planes, 1), _bn(sd, p + "bn1", planes)
        self.c2, self.b2 = _conv(sd, p + "conv2", planes, planes, 3), _bn(sd, p + "bn2", planes)
        self.pool = nn.AvgPool2d(stride) if stride > 1 else nn.Identity()
        self.c3, self.b3 = _conv(sd, p + "conv3", planes, 4 * planes, 1), _bn(sd, p + "bn3", 4 * planes)
        self.down = None
        if stride > 1 or cin != 4 * planes:
            self.down = nn.Sequential(nn.AvgPool2d(stride) if stride > 1 else nn.Identity(),
                                      _conv(sd, p + "downsample.0", cin, 4 * planes, 1),
                                      _bn(sd, p + "downsample.1", 4 * planes))
        self.relu = nn.ReLU()

    def forward(self, x):
        out = self.relu(self.b1(self.c1(x)))
        out = self.relu(self.b2(self.c2(out)))
        out = self.b3(self.c3(self.pool(out)))
        return self.relu(out + (self.down(x) if self.down is not None else x))


@torch.no_grad()
def image_features(sd, arch, px):
    w = arch.width
    stem = nn.Sequential(_conv(sd, "visual.conv1", 3, w // 2, 3, 2), _bn(sd, "visual.bn1", w // 2), nn.ReLU(),
                         _conv(sd, "visual.conv2", w // 2, w // 2, 3), _bn(sd, "visual.bn2", w // 2), nn.ReLU(),
                         _conv(sd, "visual.conv3", w // 2, w, 3), _bn(sd, "visual.bn3", w), nn.ReLU(), nn.AvgPool2d(2))
    blocks, cin = [], w
    for s, n in enumerate(arch.layers):
        for j in range(n):
            blocks.append(Bottleneck(sd, "visual.layer%d.%d." % (s + 1, j), cin, w << s, 2 if (j == 0 and s > 0) else 1))
            cin = 4 * (w << s)
    x = nn.Sequential(stem, *blocks)(px)
    # OpenAI's AttentionPool2d: (HW, B, C) tokens with the mean prepended, + positional embedding
    x = x.flatten(start_dim=2).permute(2, 0, 1)
    x = torch.cat([x.mean(dim=0, keepdim=True), x], dim=0) + sd["visual.attnpool.positional_embedding"][:, None, :]
    a = "visual.attnpool."
    C = x.shape[-1]
    out, _ = F.multi_head_attention_forward(
        query=x[:1], key=x, value=x, embed_dim_to_check=C, num_heads=C // 64,
        q_proj_weight=sd[a + "q_proj.weight"], k_proj_weight=sd[a + "k_proj.weight"], v_proj_weight=sd[a + "v_proj.weight"],
        in_proj_weight=None, in_proj_bias=torch.cat([sd[a + "q_proj.bias"], sd[a + "k_proj.bias"], sd[a + "v_proj.bias"]]),
        bias_k=None, bias_v=None, add_zero_attn=False, dropout_p=0.0,
        out_proj_weight=sd[a + "c_proj.weight"], out_proj_bias=sd[a + "c_proj.bias"],
        use_separate_proj_weight=True, training=False, need_weights=False)
    return out[0]


def main():
    sd = m.synthetic_state_dict(TINY, seed=0)
    px = clip_ref.synth_images(N, TINY)
    feats = image_features(sd, TINY, px)
    np.savez(OUT, image=feats.numpy().astype(np.float32))
    print("wrote", OUT, tuple(feats.shape))


if __name__ == "__main__":
    main()
