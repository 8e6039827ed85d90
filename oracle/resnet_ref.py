"""fp32 restatement of the ResNet CLIP image tower (OpenAI's ModifiedResNet), functional and with every BatchNorm kept
separate from its convolution (the library folds them at load time).  `sd` is a state_dict in OpenAI's key layout,
`arch` a model.ResNetArch (or anything with `layers`, `width`, `image_size`).  The text tower is oracle.clip_ref's
encode_text, which reads only arch.text and arch.quick_gelu.

  stem:   3 x (conv 3x3 pad 1 -> BN -> ReLU), the first at stride 2, then AvgPool2d(2)
  stages: Bottleneck blocks, planes width * 2^i, stride 1, 2, 2, 2:
          conv1 1x1 -> BN -> ReLU -> conv2 3x3 pad 1 -> BN -> ReLU -> AvgPool(stride) -> conv3 1x1 -> BN,
          + identity (downsample = AvgPool(stride) -> conv 1x1 -> BN when stride > 1 or cin != 4 planes), ReLU
  attnpool: tokens = [spatial mean, pixels] + positional_embedding; one query (token 0), heads of 64, c_proj.
"""
import torch
import torch.nn.functional as F

from . import clip_ref


def _bn(x, sd, p):
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"],
                        training=False, momentum=0.0, eps=1e-5)


def _conv_bn(x, sd, conv, bn, stride=1, padding=0):
    return _bn(F.conv2d(x, sd[conv + ".weight"], stride=stride, padding=padding), sd, bn)


def stem(sd, x):
    x = F.relu(_conv_bn(x, sd, "visual.conv1", "visual.bn1", stride=2, padding=1))
    x = F.relu(_conv_bn(x, sd, "visual.conv2", "visual.bn2", padding=1))
    x = F.relu(_conv_bn(x, sd, "visual.conv3", "visual.bn3", padding=1))
    return F.avg_pool2d(x, 2)


def bottleneck(sd, p, x, stride):
    out = F.relu(_conv_bn(x, sd, p + "conv1", p + "bn1"))
    out = F.relu(_conv_bn(out, sd, p + "conv2", p + "bn2", padding=1))
    if stride > 1:
        out = F.avg_pool2d(out, stride)
    out = _conv_bn(out, sd, p + "conv3", p + "bn3")
    idn = x
    if (p + "downsample.0.weight") in sd:
        if stride > 1:
            idn = F.avg_pool2d(idn, stride)
        idn = _conv_bn(idn, sd, p + "downsample.0", p + "downsample.1")
    return F.relu(out + idn)


def attnpool(sd, x, heads):
    """x [B, C, H, W] -> [B, D]: the query is the mean token only (token 0 of the full attention's output)."""
    a = "visual.attnpool."
    B, C, H, W = x.shape
    t = x.flatten(2).permute(0, 2, 1)                                  # [B, HW, C]
    t = torch.cat([t.mean(dim=1, keepdim=True), t], dim=1) + sd[a + "positional_embedding"]
    q = t[:, :1] @ sd[a + "q_proj.weight"].t() + sd[a + "q_proj.bias"]
    k = t @ sd[a + "k_proj.weight"].t() + sd[a + "k_proj.bias"]
    v = t @ sd[a + "v_proj.weight"].t() + sd[a + "v_proj.bias"]
    hd = C // heads
    q = q.view(B, 1, heads, hd).transpose(1, 2)
    k = k.view(B, -1, heads, hd).transpose(1, 2)
    v = v.view(B, -1, heads, hd).transpose(1, 2)
    o = torch.softmax((q @ k.transpose(-1, -2)) * hd ** -0.5, dim=-1) @ v   # [B, heads, 1, hd]
    o = o.transpose(1, 2).reshape(B, C)
    return o @ sd[a + "c_proj.weight"].t() + sd[a + "c_proj.bias"]


def stages(sd, arch, x):
    for s, n in enumerate(arch.layers):
        for j in range(n):
            x = bottleneck(sd, "visual.layer%d.%d." % (s + 1, j), x, 2 if (j == 0 and s > 0) else 1)
    return x


@torch.no_grad()
def encode_image(sd, arch, pixels):
    """model.encode_image: fp32 NCHW [B, 3, S, S] -> [B, D] (un-normalised)."""
    sd = {k: v.float() for k, v in sd.items()}
    x = stages(sd, arch, stem(sd, pixels.float()))
    return attnpool(sd, x, 32 * arch.width // 64)


def mapper_image(sd, arch, pixels):
    f = encode_image(sd, arch, pixels)
    return (f / f.norm(dim=-1, keepdim=True)).to(torch.float16).numpy()


def encode_text(sd, arch, tokens):
    return clip_ref.encode_text({k: v.float() for k, v in sd.items()}, arch, tokens)
