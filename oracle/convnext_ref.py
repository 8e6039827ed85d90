"""fp32 restatement of the ConvNeXt CLIP image tower (timm's ConvNeXt trunk under open_clip's head), functional, with
each block's layer scale gamma applied on its own (the library folds it into fc2 at load time).  `sd` is a state_dict
in open_clip's key layout, `arch` a model.ConvNeXtArch (or anything with `depths`, `dims`, `head_mlp`, `eps`).  The
text tower is oracle.clip_ref's encode_text, which reads only arch.text and arch.quick_gelu.

  stem:   conv 4x4 stride 4 (+ bias) -> LayerNorm over channels
  stages: for s > 0: LayerNorm -> conv 2x2 stride 2 (+ bias); then blocks:
          x + gamma * fc2(gelu(fc1(LN(dwconv7x7(x) + bias))))
  head:   mean over H, W -> LayerNorm -> proj (no bias), or fc1 (+ bias) -> gelu -> fc2 (no bias)
"""
import torch
import torch.nn.functional as F

from . import clip_ref


def ln_channels(x, sd, p, eps):
    """LayerNorm over the channels of NCHW x."""
    return F.layer_norm(x.permute(0, 2, 3, 1), (x.shape[1],), sd[p + ".weight"], sd[p + ".bias"], eps).permute(0, 3, 1, 2)


def block(sd, p, x, eps):
    C = x.shape[1]
    y = F.conv2d(x, sd[p + "conv_dw.weight"], sd[p + "conv_dw.bias"], padding=3, groups=C).permute(0, 2, 3, 1)
    y = F.layer_norm(y, (C,), sd[p + "norm.weight"], sd[p + "norm.bias"], eps)
    y = F.linear(F.gelu(F.linear(y, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"])), sd[p + "mlp.fc2.weight"],
                 sd[p + "mlp.fc2.bias"])
    return x + (y * sd[p + "gamma"]).permute(0, 3, 1, 2)


def trunk(sd, arch, x):
    """NCHW pixels -> the last stage's map [B, C3, H, W]."""
    t, eps = "visual.trunk.", arch.eps
    x = ln_channels(F.conv2d(x, sd[t + "stem.0.weight"], sd[t + "stem.0.bias"], stride=4), sd, t + "stem.1", eps)
    for s, n in enumerate(arch.depths):
        p = "%sstages.%d." % (t, s)
        if s > 0:
            x = F.conv2d(ln_channels(x, sd, p + "downsample.0", eps), sd[p + "downsample.1.weight"],
                         sd[p + "downsample.1.bias"], stride=2)
        for j in range(n):
            x = block(sd, "%sblocks.%d." % (p, j), x, eps)
    return x


def head(sd, arch, pooled):
    """The normalised pooled row [B, C3] -> features [B, D]."""
    if arch.head_mlp:
        h = F.gelu(F.linear(pooled, sd["visual.head.mlp.fc1.weight"], sd["visual.head.mlp.fc1.bias"]))
        return F.linear(h, sd["visual.head.mlp.fc2.weight"])
    return F.linear(pooled, sd["visual.head.proj.weight"])


@torch.no_grad()
def encode_image(sd, arch, pixels):
    """model.encode_image: fp32 NCHW [B, 3, S, S] -> [B, D] (un-normalised)."""
    sd = {k: v.float() for k, v in sd.items()}
    x = trunk(sd, arch, pixels.float()).mean((2, 3))
    t = "visual.trunk.head.norm"
    return head(sd, arch, F.layer_norm(x, (x.shape[1],), sd[t + ".weight"], sd[t + ".bias"], arch.eps))


def encode_text(sd, arch, tokens):
    return clip_ref.encode_text({k: v.float() for k, v in sd.items()}, arch, tokens)
