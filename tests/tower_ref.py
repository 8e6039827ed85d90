"""A float64 forward of both CLIP towers that stores what the CUDA forward (csrc/clip_model.cu) stores, and the rounding
envelope the tower parity tests (test_tower_parity_cpu.py, test_tower_parity_gpu.py) accept a result under.

What it emulates is the stored data, not the arithmetic order:
  weights   as the handle holds them after b200_clip_load_weights: bf16 (round to nearest even from the fp32 state_dict)
            for every GEMM weight, `visual.conv1.weight`, `visual.positional_embedding` (the patch GEMM's residual),
            `token_embedding.weight`, `visual.proj` and `text_projection`; fp32 for the LayerNorm affine, the biases,
            the text `positional_embedding` and the class row `class_embedding + positional_embedding[0]` (summed in
            fp32 by the loader);
  stores    bf16 at every point where the forward writes bf16: `cols` after im2col; `x` after the patch GEMM + positional
            residual and the class rows; `x` after the in-place ln_pre; the text `x` after token + positional embedding;
            per layer h, qkv, the attention output a, x, h, f, x; and inside the attention kernels, the unnormalised
            probabilities exp(s - max) before P.V (normalised afterwards by the sum of the unrounded ones);
  tail      pooled LayerNorm and projection in float64 (the kernel keeps them in fp32, embed_kernels_ref.py bounds that
            error, which is far below a bf16 step), then features / |features| and the fp16 or fp32 cast of
            pool_ln_proj_norm.
Everything between two store points is float64.

`rounding` picks what a store point does: "nearest" gives y_RN, the forward of exactly rounded stores; ("directed",
seed) sends each stored element to its lower or upper bf16 neighbour, chosen at random.

The envelope of one output row is E = max over S_DIRECTED directed runs of |y_s - y_RN|_2, and a row of raw features y
is accepted when |y - y_RN|_2 <= 2 E.  This is not a proof.  A correct GPU forward differs from y_RN only where its
fp32 value of a stored element lands on the other bf16 neighbour than the exact value does (and, in the softmax, where
its running maximum rounds the probabilities at another scale): a sparse subset of the elements that every directed
run moves, by at most the same step.  The factor of 2 is justified by test_tower_parity_cpu.py, not derived: an fp32
implementation with the same stores (another summation order, and the kernels' running-maximum softmax) stays well
inside it on every case, and each named wrong forward lands outside it, most by ten times or more.

Cases: one per distinct (architecture, activation) of model.ARCHS (the "ViT-H/14" alias is the open_clip:ViT-H-14
entry), at every real shape (width, heads, mlp, tokens, patch, image size, embed_dim, activation) but with
LAYERS = 2 blocks per tower: enough to catch a layer's weights indexed wrongly, cheap enough for a float64 oracle.
Weights come from oracle.clip_ref.make_state_dict, as is and sensitised (WEIGHTS).  Samples are independent, so the oracle runs on single samples,
and each sample of a batch is regenerated from its own seed (image_input / text_input)."""
import functools
import math

import torch

from oracle import clip_ref

LAYERS = 2
S_DIRECTED = 8
ACCEPT = 2.0                      # |y - y_RN| <= ACCEPT * E
LN_EPS = 1e-5
COS_TOL = 1e-3                    # the older tower tests' bound on 1 - cos (test_embed_gpu.py)

# The wrong forwards of test_tower_parity_cpu.py, and the towers each one applies to.
MUTATIONS = {
    "act_swapped": ("image", "text"),        # quick-GELU <-> erf GELU
    "no_causal_mask": ("text",),
    "pos_shifted": ("image",),               # positional row p instead of 1 + p for patch p (res_row_off = 0)
    "ln_pre_skipped": ("image",),
    "layer1_with_layer0": ("image", "text"),  # the second block runs with the first block's weights
    "scale_from_width": ("image", "text"),   # softmax scale w^-0.5 instead of head_dim^-0.5
    "eot_one_early": ("text",),              # pooled row argmax(tokens) - 1
}


# ---- cases ------------------------------------------------------------------------------------------------------

def _case_name(arch):
    import clip_retrieval_b200 as m

    return next(k for k, a in m.ARCHS.items() if a == arch)


def cases():
    """name -> model.ClipArch (all LAYERS deep): one per distinct ARCHS value, named by its first key."""
    import clip_retrieval_b200 as m
    from dataclasses import replace

    out = {}
    for a in m.ARCHS.values():
        name = _case_name(a)
        out[name] = replace(a, vision=replace(a.vision, layers=LAYERS), text=replace(a.text, layers=LAYERS))
    return out


def case_of(key):
    """The case an ARCHS key is checked by."""
    import clip_retrieval_b200 as m

    return _case_name(m.ARCHS[key])


def clip_cfg(arch):
    """The oracle.clip_ref config of a case (its weights come from clip_ref.make_state_dict)."""
    t = lambda tw: clip_ref.TowerCfg(tw.width, tw.layers, tw.heads, tw.mlp)   # noqa: E731
    return clip_ref.ClipCfg(arch.embed_dim, arch.image_size, arch.patch, t(arch.vision), t(arch.text),
                            arch.context_length, arch.vocab_size, arch.quick_gelu)


# Two weight sets per case.  "plain" is clip_ref.make_state_dict's initialisation (seed 0).  Under it three wrong
# forwards hide inside the bf16 store noise: the pre-activations of c_fc (std ~0.7 around 0) sit where quick-GELU and
# erf GELU differ by ~1 %; near-uniform attention averages the positional rows of all patches, so rows shifted by one
# nearly cancel; and a softmax of near-zero scores barely changes with its scale.  "sensitised" moves the weights into
# the regime where those errors show (trained CLIPs have peaked attention and large positional tables too), at the
# price of a noisier envelope for the other wrong forwards, which the plain set keeps far outside it.
WEIGHTS = ("plain", "sensitised")
POS_SCALE = 20.0        # visual.positional_embedding (and so the class row): std 20 w^-0.5, comparable to the patches
QK_SCALE = 3.0          # the q and k rows of in_proj (weight and bias): scores 9x larger, attention far from uniform
FC_BIAS_SHIFT = -2.0    # c_fc bias: pre-activations around -2, where the two GELUs differ by a large part of the value
PROJ_SCALE = 8.0        # c_proj weight: the MLP branch carries that difference into the residual stream


def sensitise(sd):
    """The state_dict with POS_SCALE, QK_SCALE, FC_BIAS_SHIFT and PROJ_SCALE applied."""
    sd = dict(sd)
    for k in list(sd):
        if k.endswith(("attn.in_proj_weight", "attn.in_proj_bias")):
            t = sd[k].clone()
            t[:2 * (t.shape[0] // 3)] *= QK_SCALE
            sd[k] = t
        elif k.endswith("mlp.c_fc.bias"):
            sd[k] = sd[k] + FC_BIAS_SHIFT
        elif k.endswith("mlp.c_proj.weight"):
            sd[k] = sd[k] * PROJ_SCALE
    sd["visual.positional_embedding"] = sd["visual.positional_embedding"] * POS_SCALE
    return sd


@functools.lru_cache(maxsize=2)
def state_dict(name, weights="plain"):
    """clip_ref.make_state_dict of the case (seed 0), sensitised when weights == "sensitised"."""
    if weights not in WEIGHTS:
        raise ValueError("weights %r: one of %s" % (weights, WEIGHTS))
    sd = clip_ref.make_state_dict(clip_cfg(cases()[name]), seed=0)
    return sensitise(sd) if weights == "sensitised" else sd


def image_tokens(arch):
    return (arch.image_size // arch.patch) ** 2 + 1


# ---- inputs: each sample from its own seed ------------------------------------------------------------------------

def image_input(arch, i):
    """Sample i: fp32 [3, S, S] in the range of the real preprocess output."""
    g = torch.Generator().manual_seed(31337 + 7919 * i + arch.image_size)
    return torch.randn(3, arch.image_size, arch.image_size, generator=g).clamp_(-1.80, 2.15)


TEXT_KINDS = ("random length", "full length", "EOT at 1", "EOT twice")


def text_input(arch, i):
    """Sample i: int64 [T] of kind TEXT_KINDS[i % 4]: SOT, ids < SOT, EOT (the largest id), zero padding.  "full
    length" fills every position; "EOT at 1" pools row 1; "EOT twice" holds a second EOT after the first (the first
    maximum is the pooled row)."""
    g = torch.Generator().manual_seed(4242 + 7919 * i)
    T, sot, eot = arch.context_length, arch.vocab_size - 2, arch.vocab_size - 1
    ids = lambda n: torch.randint(1, sot, (n,), generator=g)   # noqa: E731
    row = torch.zeros(T, dtype=torch.int64)
    row[0] = sot
    kind = TEXT_KINDS[i % 4]
    if kind == "random length":
        n = int(torch.randint(1, T - 1, (1,), generator=g))
        row[1:1 + n], row[1 + n] = ids(n), eot
    elif kind == "full length":
        row[1:T - 1], row[T - 1] = ids(T - 2), eot
    elif kind == "EOT at 1":
        row[1] = eot
    else:
        a = int(torch.randint(2, T // 2, (1,), generator=g))
        b = int(torch.randint(a + 1, T, (1,), generator=g))
        row[1:b] = ids(b - 1)
        row[a], row[b] = eot, eot
    return row


def sample(arch, tower, i):
    return image_input(arch, i) if tower == "image" else text_input(arch, i)


def batch(arch, tower, n, first=0):
    return torch.stack([sample(arch, tower, i) for i in range(first, first + n)])


# ---- float64 -> bf16 in one rounding ------------------------------------------------------------------------------

def round_bf16(x, rounding="nearest", gen=None):
    """x rounded to a bf16 value (returned as float64) in a single step from float64: x = q * ulp exactly, with
    ulp = 2^(e - 8) for x in [2^(e-1), 2^e) (8 significant bits; subnormal spacing 2^-133 below 2^-126), and q rounded
    to an integer: half to even ("nearest"), or down or up at random ("directed", gen draws the choice).  A cast
    through float32 would round twice."""
    x = x.double()
    _, e = torch.frexp(x)
    ulp = torch.ldexp(torch.ones_like(x), e.clamp(min=-125) - 8)
    q = x / ulp
    if rounding == "nearest":
        r = torch.round(q)
    else:
        lo = torch.floor(q)
        up = torch.rand(q.shape, generator=gen, device=q.device, dtype=torch.float64) < 0.5
        r = torch.where(q == lo, lo, lo + up.double())
    return r * ulp


def _rounder(rounding, device, dtype):
    if rounding == "nearest":
        return lambda t: round_bf16(t).to(dtype)
    kind, seed = rounding
    if kind != "directed":
        raise ValueError("rounding %r: 'nearest' or ('directed', seed)" % (rounding,))
    gen = torch.Generator(device=device).manual_seed(int(seed))
    return lambda t: round_bf16(t, "directed", gen).to(dtype)


# ---- the handle's weights -------------------------------------------------------------------------------------------

def handle_weights(sd, device, dtype=torch.float64):
    """The state_dict as b200_clip_load_weights stores it (see the module docstring), as `dtype` tensors."""
    bf = lambda k: sd[k].float().bfloat16().to(device, dtype)   # noqa: E731  (fp32 -> bf16: one RN step)
    f32 = lambda k: sd[k].float().to(device, dtype)             # noqa: E731
    W = {}
    for k in sd:
        if k.endswith(("in_proj_weight", "out_proj.weight", "c_fc.weight", "c_proj.weight")):
            W[k] = bf(k)
        elif k.endswith(("ln_1.weight", "ln_1.bias", "ln_2.weight", "ln_2.bias", "in_proj_bias", "out_proj.bias",
                         "c_fc.bias", "c_proj.bias")):
            W[k] = f32(k)
    for k in ("visual.positional_embedding", "token_embedding.weight", "visual.proj", "text_projection"):
        W[k] = bf(k)
    for k in ("visual.ln_pre.weight", "visual.ln_pre.bias", "visual.ln_post.weight", "visual.ln_post.bias",
              "ln_final.weight", "ln_final.bias", "positional_embedding"):
        W[k] = f32(k)
    cw = sd["visual.conv1.weight"]
    W["visual.conv1.weight"] = cw.reshape(cw.shape[0], -1).float().bfloat16().to(device, dtype)
    W["cls_pos0"] = (sd["visual.class_embedding"].float() + sd["visual.positional_embedding"][0].float()).to(device, dtype)
    return W


# ---- the forward ----------------------------------------------------------------------------------------------------

def _ln(x, g, b):
    mu = x.mean(-1, keepdim=True)
    d = x - mu
    return d * torch.rsqrt((d * d).mean(-1, keepdim=True) + LN_EPS) * g + b


def _act(x, quick):
    return x * torch.sigmoid(1.702 * x) if quick else 0.5 * x * (1.0 + torch.erf(x * 0.5 ** 0.5))


def _attention(qkv, heads, causal, rnd, scale_from_width):
    """softmax(Q K^T hd^-0.5 [+ causal mask]) V of one sample's stored qkv [T, 3w], with the probabilities taken from
    test_embed_gpu.attention_ref64 (its float64 model of the kernels) and stored as bf16 before P.V."""
    from test_embed_gpu import attention_ref64

    T, w = qkv.shape[0], qkv.shape[1] // 3
    hd = w // heads
    src = qkv
    if scale_from_width:
        src = qkv.clone()
        src[:, :w] *= (hd / w) ** 0.5
    v = qkv[:, 2 * w:].view(T, heads, hd).transpose(0, 1)
    if qkv.dtype != torch.float64:
        return _attention_online(src, v, heads, hd, causal, rnd).transpose(0, 1).reshape(T, w)
    _, _, P = attention_ref64(src, 1, T, heads, hd, causal)
    e = (P[0] / P[0].amax(-1, keepdim=True))            # exp(s - max): what the kernels round before P.V
    a = (rnd(e) @ v) / e.sum(-1, keepdim=True).to(qkv.dtype)
    return a.transpose(0, 1).reshape(T, w)


def _attention_online(qkv, v, heads, hd, causal, rnd, block=64):
    """The fp32 stand-in's attention, run as the kernels run it: scores in qkv.dtype, keys in blocks of 64 under a
    running maximum m, exp(s - m) stored as bf16 before P.V at the scale of the m current for its block, the
    accumulator and the sum of the unrounded exponentials rescaled when m grows."""
    T, w = qkv.shape[0], qkv.shape[1] // 3
    q = qkv[:, :w].view(T, heads, hd).transpose(0, 1)
    k = qkv[:, w:2 * w].view(T, heads, hd).transpose(0, 1)
    s = (q @ k.transpose(-1, -2)) * hd ** -0.5
    if causal:
        s = s.masked_fill(torch.ones(T, T, dtype=torch.bool, device=s.device).triu_(1), float("-inf"))
    m = torch.full((heads, T, 1), float("-inf"), dtype=s.dtype, device=s.device)
    acc = torch.zeros(heads, T, hd, dtype=s.dtype, device=s.device)
    tot = torch.zeros(heads, T, 1, dtype=s.dtype, device=s.device)
    for k0 in range(0, T, block):
        sb = s[:, :, k0:k0 + block]
        m_new = torch.maximum(m, sb.amax(-1, keepdim=True))
        alpha = torch.exp(m - m_new).nan_to_num(0.0)        # rows whose keys so far are all masked keep nothing
        p = torch.exp(sb - m_new).nan_to_num(0.0)
        acc = acc * alpha + rnd(p) @ v[:, k0:k0 + block]
        tot = tot * alpha + p.sum(-1, keepdim=True)
        m = m_new
    return acc / tot


def _block(x, W, p, heads, quick, causal, rnd, mutation):
    h = rnd(_ln(x, W[p + "ln_1.weight"], W[p + "ln_1.bias"]))
    qkv = rnd(h @ W[p + "attn.in_proj_weight"].t() + W[p + "attn.in_proj_bias"])
    a = rnd(_attention(qkv, heads, causal, rnd, mutation == "scale_from_width"))
    x = rnd(a @ W[p + "attn.out_proj.weight"].t() + W[p + "attn.out_proj.bias"] + x)
    h = rnd(_ln(x, W[p + "ln_2.weight"], W[p + "ln_2.bias"]))
    f = rnd(_act(h @ W[p + "mlp.c_fc.weight"].t() + W[p + "mlp.c_fc.bias"], quick))
    return rnd(f @ W[p + "mlp.c_proj.weight"].t() + W[p + "mlp.c_proj.bias"] + x)


def forward(W, arch, tower, inp, rounding="nearest", dtype=torch.float64, mutation=None):
    """Raw features [D] (float64) of one sample: pixels [3, S, S] (tower "image") or tokens [T] ("text").
    dtype is the arithmetic between stores (float64 for the oracle; float32 gives the stand-in of the CPU tests, with
    W from handle_weights(..., dtype=torch.float32)).  mutation: None or a MUTATIONS key, for the CPU tests."""
    dev = W["cls_pos0"].device
    rnd = _rounder(rounding, dev, dtype)
    quick = arch.quick_gelu != (mutation == "act_swapped")
    if tower == "image":
        t, pre = arch.vision, "visual."
        p, g, w = arch.patch, arch.image_size // arch.patch, arch.vision.width
        cols = rnd(inp.to(dev, dtype).view(3, g, p, g, p).permute(1, 3, 0, 2, 4).reshape(g * g, 3 * p * p))
        off = 0 if mutation == "pos_shifted" else 1
        patches = rnd(cols @ W["visual.conv1.weight"].t() + W["visual.positional_embedding"][off:off + g * g])
        x = torch.cat([rnd(W["cls_pos0"])[None], patches])
        if mutation != "ln_pre_skipped":
            x = rnd(_ln(x, W["visual.ln_pre.weight"], W["visual.ln_pre.bias"]))
        causal, pool = 0, 0
    else:
        t, pre = arch.text, ""
        tok = inp.to(dev)
        x = rnd(W["token_embedding.weight"][tok] + W["positional_embedding"][:tok.shape[0]])
        causal = 0 if mutation == "no_causal_mask" else 1
        pool = int(torch.argmax(tok)) - (1 if mutation == "eot_one_early" else 0)
    for i in range(t.layers):
        li = 0 if (mutation == "layer1_with_layer0" and i == 1) else i
        x = _block(x, W, "%stransformer.resblocks.%d." % (pre, li), t.heads, quick, causal, rnd, mutation)
    lnf = ("visual.ln_post." if tower == "image" else "ln_final.")
    z = _ln(x[pool], W[lnf + "weight"], W[lnf + "bias"])
    return (z @ W["visual.proj" if tower == "image" else "text_projection"]).double()


# ---- the envelope -----------------------------------------------------------------------------------------------------

def envelope(W, arch, tower, inp):
    """(y_RN [D] float64, E): the forward with nearest stores and the largest distance of S_DIRECTED directed runs
    from it."""
    y = forward(W, arch, tower, inp)
    E = max(float((forward(W, arch, tower, inp, ("directed", s)) - y).norm()) for s in range(S_DIRECTED))
    return y, E


def feature_ratio(got, y_rn, E):
    """|got - y_RN|_2 / (ACCEPT E) for raw fp32 features: accepted when <= 1."""
    return float((got.double().to(y_rn.device) - y_rn).norm()) / (ACCEPT * E)


def ulp_f16(x):
    """The fp16 spacing at |x| (2^-24 below the normal range)."""
    _, e = torch.frexp(x.double().abs())
    return torch.ldexp(torch.ones_like(x, dtype=torch.float64), e.clamp(min=-13) - 11)


def normalised_ratio(got, y_rn, E):
    """|got - n|_2 / bound for a normalised output row (fp16 or fp32) against n = y_RN / |y_RN|.

    Derivation.  Let f be the forward's raw features, accepted as |f - y_RN| <= 2E.  For any u, v != 0,
    |u/|u| - v/|v|| <= |u - v|/|v| + ||v| - |u||/|v| <= 2|u - v|/|v|, so |f/|f| - n| <= 4E/|y_RN|.  The fp32
    normalisation (a sum of D squares, sqrtf, a reciprocal, a product) moves each element by a few fp32 ulps, under
    2^-20 in norm for a unit row.  The fp16 cast moves element j by at most half an fp16 ulp of the value it rounds,
    which lies within the two terms above of n_j and so within one ulp of n_j's binade: |cast| <= |ulp16(n)|_2.
        bound = 4E / |y_RN| + 2^-20 + |ulp16(n)|_2   (the last term only for fp16 outputs)."""
    n = y_rn / y_rn.norm()
    bound = 2 * ACCEPT * E / float(y_rn.norm()) + 2.0 ** -20
    if got.dtype == torch.float16:
        bound += float(ulp_f16(n).norm())
    return float((got.double().to(n.device) - n).norm()) / bound


def cosine_distance(got, y_rn):
    """1 - cos(got, y_RN): the quantity the older tower tests hold under COS_TOL."""
    g = got.double().to(y_rn.device)
    return 1.0 - float(g @ y_rn) / float(g.norm() * y_rn.norm())
