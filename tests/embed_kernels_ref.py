"""Cases and float64 references with per-element error bounds for the embed path's non-GEMM kernels (LayerNorm, the
vision and text tower fronts, the pooled LN -> projection -> normalise end, the masked-mean linear head).

The cases come from the model tables (`model.ARCHS`, `mclip.MCLIP_ARCHS`, `xlmr_clip.XLMR_CLIP_ARCHS`), so a new
architecture is covered as soon as it is added.  The bounds are shared by the GPU parity tests
(test_embed_kernels_gpu.py), which compare the kernels with them, and the CPU tests (test_embed_kernels_cpu.py), which
show that each bound rejects named wrong kernels.

Notation: u = 2^-24 (fp32 unit roundoff), gamma(n) = n u / (1 - n u) bounds n roundings along one chain, a bf16 store
adds 2^-8 relative and an fp16 store 2^-11 relative (plus 2^-25 absolute below fp16's normal range).  rsqrtf is within
2 ulp (4u); sqrtf and `/` are correctly rounded (the library is built without fast math)."""
import math

import torch

U = 2.0 ** -24
U_BF16 = 2.0 ** -8
U_F16 = 2.0 ** -11
TINY = 1e-30

# Every template instantiation of layernorm_kernel<CPL> (16-byte chunks per lane, CPL = ceil(w / 256)): a width at
# each CPL's low and high end, 200 (a partial last chunk round), 264 (CPL 2 with one live chunk in the second round).
LN_TEMPLATE_WIDTHS = (8, 64, 200, 256, 264, 512, 768, 1024, 1280, 1536, 1792, 2048)
# Warps of the persistent LayerNorm grid (132 x 6 blocks of 8 warps): rows past it go round the strided loop that
# prefetches the next row.
LN_PERSISTENT_ROWS = 132 * 6 * 8
LN_EDGE_ROWS = (1, 7, 8, LN_PERSISTENT_ROWS - 1, LN_PERSISTENT_ROWS, LN_PERSISTENT_ROWS + 1, 2 * LN_PERSISTENT_ROWS + 1)
LN_EPS = (1e-5, 1e-12)
# Row classes of layernorm_inputs, by row % 5.
LN_CLASSES = ("ordinary", "large mean", "variance ~ 1e-5", "variance ~ 1e-12", "constant")


def gamma(n):
    return n * U / (1 - n * U)


def within(out, ref, bound):
    """True when every |out - ref| <= bound (a NaN anywhere is a failure)."""
    return bool(((out.double() - ref).abs() <= bound).all())


def assert_within(out, ref, bound, what=""):
    err = (out.double() - ref).abs()
    ok = err <= bound
    if not bool(ok.all()):
        bad = (~ok).nonzero()[0].tolist()
        raise AssertionError("%s: %d elements out of bound, first at %s: got %r want %r bound %r (max err / bound %g)"
                             % (what, int((~ok).sum()), bad, float(out.double()[tuple(bad)]), float(ref[tuple(bad)]),
                                float(bound[tuple(bad)]), float(torch.nan_to_num(err / bound, nan=float("inf")).max())))


# ---- the model tables -> cases ----------------------------------------------------------------------------------

def vision_tokens(a):
    return (a.image_size // a.patch) ** 2 + 1


def clip_archs():
    """name -> model.ClipArch of every CLIP the library serves, the image towers of the XLM-R CLIPs included (their
    text width is 0: no CLIP text tower)."""
    import clip_retrieval_b200 as m
    from clip_retrieval_b200 import xlmr_clip

    out = dict(m.ARCHS)
    out.update({"xlmr:" + k: a.vision for k, a in xlmr_clip.XLMR_CLIP_ARCHS.items()})
    return out


def encoder_archs():
    """name -> mclip.EncoderArch of every BERT-family text tower (M-CLIP and the XLM-R CLIPs)."""
    from clip_retrieval_b200 import mclip, xlmr_clip

    out = dict(mclip.MCLIP_ARCHS)
    out.update({"xlmr:" + k: a.text for k, a in xlmr_clip.XLMR_CLIP_ARCHS.items()})
    return out


def tiny_clip_configs():
    """The oracle's small CLIP configs (tile tails, other patch sizes)."""
    from oracle import clip_ref

    return {k: c for k, c in clip_ref.CONFIGS.items() if k.startswith("tiny")}


def layernorm_cases():
    """(w, rows): every template width at the edge row counts of the persistent grid, then each tower of the tables at
    a serving batch (B T rows: 256 samples, 64 past 300 tokens)."""
    cases = [(w, r) for w in LN_TEMPLATE_WIDTHS for r in LN_EDGE_ROWS]
    for a in clip_archs().values():
        T = vision_tokens(a)
        cases.append((a.vision.width, (256 if T <= 300 else 64) * T))
        if a.text.width:
            cases.append((a.text.width, 256 * a.context_length))
    for e in encoder_archs().values():
        cases.append((e.width, 64 * 77))
    return sorted(set(cases))


def im2col_cases():
    """(S, p, w): image size, patch and vision width of every table CLIP and the tiny configs."""
    cases = {(a.image_size, a.patch, a.vision.width) for a in clip_archs().values()}
    cases |= {(c.image_size, c.patch, c.vision.width) for c in tiny_clip_configs().values()}
    return sorted(cases)


def text_embed_cases():
    """(w, T, vocab) of every CLIP text tower of the tables and the tiny configs."""
    cases = {(a.text.width, a.context_length, a.vocab_size) for a in clip_archs().values() if a.text.width}
    cases |= {(c.text.width, c.context_length, c.vocab_size) for c in tiny_clip_configs().values()}
    return sorted(cases)


# off-table pooled projections: D not a multiple of 64, w = 200 (a partial 256-column round of the LN)
POOL_EXTRA = ((200, 100, 5), (768, 130, 3))


def pool_cases():
    """(w, D, T): the vision end (w, embed_dim, image tokens) and the text end (w, embed_dim, context length) of
    every table CLIP, and POOL_EXTRA."""
    cases = set(POOL_EXTRA)
    for a in clip_archs().values():
        cases.add((a.vision.width, a.embed_dim, vision_tokens(a)))
        if a.text.width:
            cases.add((a.text.width, a.embed_dim, a.context_length))
    return sorted(cases)


# off-table masked-mean heads: the XLM-R-base CLIP head's hidden width as D, and a small odd shape
MEAN_PROJ_EXTRA = ((1024, 640), (200, 100))


def mean_proj_cases():
    """(w, D) of every M-CLIP linear head, and MEAN_PROJ_EXTRA.  Each runs with and without a bias."""
    from clip_retrieval_b200 import mclip

    return sorted({(e.width, e.out_dim) for e in mclip.MCLIP_ARCHS.values()} | set(MEAN_PROJ_EXTRA))


# ---- inputs -----------------------------------------------------------------------------------------------------

def layernorm_inputs(rows, w, seed, device):
    """bf16 x [rows, w] with row classes by row % 5 (LN_CLASSES): N(0.5, 3^2); 100 + N(0, 1) (a large mean over a
    small spread: cancellation in the two-pass statistics); std ~ sqrt(1e-5) and ~ sqrt(1e-12) near 0 (variance
    comparable to either epsilon); a constant row.  gamma, beta fp32 N(0, 1).  -> x, gamma, beta, class [rows]."""
    g = torch.Generator(device=device).manual_seed(seed)
    n = torch.randn(rows, w, device=device, generator=g)
    cls = torch.arange(rows, device=device) % 5
    scale = torch.tensor([3.0, 1.0, 1e-5 ** 0.5, 1e-6, 0.0], device=device)[cls][:, None]
    shift = torch.tensor([0.5, 100.0, 0.3 * 1e-5 ** 0.5, 0.3e-6, 0.0], device=device)[cls][:, None]
    const = torch.randn(rows, 1, device=device, generator=g) * (cls[:, None] == 4)
    x = (n * scale + shift + const).bfloat16()
    ga = torch.randn(w, device=device, generator=g)
    be = torch.randn(w, device=device, generator=g)
    return x, ga, be, cls


# ---- LayerNorm ----------------------------------------------------------------------------------------------------

def layernorm_depths(w, kernel):
    """(n_mean, n_var): roundings along the longest chain of the mean (sum, division) and of the variance (difference,
    square, sum, division, + eps, eps itself rounded to fp32).
      "rows" (layernorm_kernel, one warp per row): a lane adds its 4 CPL bf16 pairs (pair sum, then into the running
             sum: 4 CPL + 1), then 5 butterfly steps; its squares go through 8 CPL adds and the 5 steps.
      "pool" (pool_proj_split_kernel, one block per row): a thread adds ceil(w / 256) strided values, then 5 butterfly
             steps and 8 warp partials in sequence."""
    c = math.ceil(w / 256)
    if kernel == "rows":
        return 4 * c + 7, 8 * c + 10
    if kernel == "pool":
        return c + 14, c + 18
    raise ValueError(kernel)


def layernorm_bound(x, ga, be, eps, kernel, store_bf16=True, variance_divisor=None):
    """float64 LayerNorm of the bf16 rows x with fp32 gamma, beta, and a per-element bound on |kernel - ref|.

    mean:  |mu^ - mu| <= e_mu = gamma(n_mean) mean|x|.
    var:   sum (x - mu^)^2 = w (var + (mu^ - mu)^2) exactly, and every term is positive, so
           V^ = (var + e_mu^2 + eps)(1 + theta), |theta| <= gamma(n_var), and V^ / V - 1 <= e_V = (e_mu^2 / V)(1 +
           gamma) + gamma with V = var + eps.
    rstd:  rsqrtf(V^) / rsqrt(V) - 1 <= e_r = (1 - e_V)^-1/2 (1 + 4u) - 1 (unbounded when e_V >= 1/2).
    out:   ((x - mu^) rstd^) gamma + beta in three roundings and one add:
           |y^ - y| <= E = E1 + u (|y| + E1), E1 = |gamma| rstd (e_mu + (|x - mu| + e_mu)((1 + e_r)(1 + u)^3 - 1)),
           then the bf16 store (store_bf16) adds 2^-8 (|y| + E).
    variance_divisor (w by default) exists for the wrong variants of the CPU tests."""
    xd, g, b = x.double(), ga.double(), be.double()
    w = xd.shape[-1]
    n_mean, n_var = layernorm_depths(w, kernel)
    mu = xd.mean(-1, keepdim=True)
    d = xd - mu
    var = (d * d).sum(-1, keepdim=True) / (variance_divisor or w)
    V = var + eps
    r = V.rsqrt()
    y = d * r * g + b
    e_mu = gamma(n_mean) * xd.abs().mean(-1, keepdim=True)
    th = gamma(n_var)
    e_V = (e_mu * e_mu / V) * (1 + th) + th
    e_r = torch.where(e_V < 0.5, (1 - e_V.clamp(max=0.5)).rsqrt() * (1 + 4 * U) - 1, torch.full_like(e_V, math.inf))
    E1 = g.abs() * r * (e_mu + (d.abs() + e_mu) * ((1 + e_r) * (1 + U) ** 3 - 1))
    E = E1 + U * (y.abs() + E1)
    if store_bf16:
        E = E + U_BF16 * (y.abs() + E)
    return y, E + TINY


# ---- normalise and store ------------------------------------------------------------------------------------------

def normalise_bound(f, e, D, out_f16, normalize, zero_to_one=False):
    """ref and bound of the stored row f^ / |f^| (or f^) given the float64 features f [B, D] and |f^ - f| <= e.

    The sum of squares passes through at most ceil(D / 256) + 14 roundings (a square, ceil(D / 256) strided adds, 5
    butterfly steps, 8 warp partials); sqrtf, the reciprocal or division and the scaling add at most 3 more:
    nu = gamma(ceil(D / 256) + 14) + 4u relative.  With n = |f|, |e| the 2-norm of e and lo = n - |e|:
        |f^_j / |f^| - f_j / n| <= (e_j + |f_j| |e| / n) / lo,
    so bound_j = (e_j + |f_j| |e| / n + nu (|f_j| + e_j)) / lo (unbounded when lo <= 0).  fp16 stores add
    2^-11 (|ref| + bound) + 2^-25.  zero_to_one: a zero row divides by 1 (clip_back's normalized()), else by 0."""
    if normalize:
        n = f.norm(dim=-1, keepdim=True)
        if zero_to_one:
            n = torch.where(n == 0, torch.ones_like(n), n)
        ne = e.norm(dim=-1, keepdim=True)
        lo = n - ne
        nu = gamma(math.ceil(D / 256) + 14) + 4 * U
        ref = f / n
        bound = (e + f.abs() * ne / n + nu * (f.abs() + e)) / lo
        bound = torch.where(lo > 0, bound, torch.full_like(bound, math.inf))
    else:
        ref, bound = f, e
    if out_f16:
        bound = bound + U_F16 * (ref.abs() + bound) + 2.0 ** -25
    return ref, bound + TINY


# ---- pooled LN -> projection -> normalise ---------------------------------------------------------------------------

def pool_ln_proj_bound(z, ga, be, proj, out_f16, normalize, gamma_off=False):
    """The tower end on the pooled bf16 rows z [B, w]: LN (eps 1e-5, kept in fp32: no bf16 store) -> @ proj (bf16
    [w, D]) -> normalise -> store.  -> (feat ref, feat bound, out ref, out bound).
    The projection of a column is 4 quarters of ceil(w / 4) rows, each two interleaved fma chains, added in a tree:
    a product passes through at most ceil(w / 8) + 4 roundings, so with |z^ - z| <= E_z
        |f^ - f| <= e_f = gamma(ceil(w / 8) + 4) (|z| + E_z) @ |P| + E_z @ |P|.
    gamma_off (an LN without its scale) exists for the wrong variants of the CPU tests."""
    w, D = proj.shape
    zr, E_z = layernorm_bound(z, torch.ones_like(ga) if gamma_off else ga, be, 1e-5, "pool", store_bf16=False)
    P = proj.double()
    f = zr @ P
    e_f = gamma(math.ceil(w / 8) + 4) * ((zr.abs() + E_z) @ P.abs()) + E_z @ P.abs()
    ref, bound = normalise_bound(f, e_f, D, out_f16, normalize)
    return f, e_f, ref, bound


# ---- masked mean -> projection (+ bias) -> normalized() ---------------------------------------------------------------

def masked_mean_proj_bound(x, lengths, projT, bias, out_f16, normalize, length_offset=0):
    """The M-CLIP head on bf16 x [B, T, w] (rows t >= len[b] may hold anything, NaN included): L = clamp(len, 1, T),
    m = mean of rows t < L -> @ projT (fp32 [w, D]) (+ bias) -> normalized() -> store.
    -> (feat ref, feat bound, out ref, out bound).
      mean:  an fp32 sum of L terms in order, then a division: |m^ - m| <= e_m = gamma(L) mean_t |x|;
      proj:  e_1 = gamma(ceil(w / 8) + 4) (|m| + e_m) @ |W| + e_m @ |W| (see pool_ln_proj_bound);
      bias:  one more add: e_f = e_1 + u (|f| + e_1).
    length_offset (averaging over len + k rows) exists for the wrong variants of the CPU tests."""
    B, T, w = x.shape
    D = projT.shape[1]
    L = (lengths.clamp(1, T) + length_offset).to(torch.float64)[:, None]
    live = (torch.arange(T, device=x.device)[None, :] < L)[:, :, None]
    xd = torch.where(live, x.double(), torch.zeros((), dtype=torch.float64, device=x.device))
    m = xd.sum(1) / L
    e_m = torch.tensor([gamma(int(n)) for n in L[:, 0].tolist()], dtype=torch.float64, device=x.device)[:, None] * (
        xd.abs().sum(1) / L)
    W = projT.double()
    f = m @ W
    e_f = gamma(math.ceil(w / 8) + 4) * ((m.abs() + e_m) @ W.abs()) + e_m @ W.abs()
    if bias is not None:
        f = f + bias.double()
        e_f = e_f + U * (f.abs() + e_f)
    ref, bound = normalise_bound(f, e_f + TINY, D, out_f16, normalize, zero_to_one=True)
    return f, e_f + TINY, ref, bound
