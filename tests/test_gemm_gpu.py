"""wgmma GEMM core (csrc/gemm.cuh) against a float64 reference of the same operation, computed from the exact bf16
operands the kernel received.

Error bound, per element (y = the float64 result, x = the pre-activation value A.W^T + bias, R = the residual):

  |out - y| <= 2^-8 (|y| + e)  +  e,      e = 1.2 * acc  +  act  +  2^-22 (|x| + |R|)

- 2^-8 |y|: the bf16 store rounds to nearest; bf16 keeps 8 significant bits, so half an ulp is at most 2^-8 of the
  value.
- acc = (ceil(K / 16) + 2) * 2^-22 * S,  S = |A| . |W|^T:  bf16 x bf16 products are exact in fp32.  Each wgmma k16
  step adds 16 of them to the fp32 accumulator; we allow one fp32 ulp (2^-23, truncation, not just rounding) of
  the partial sum's magnitude <= S per step, twice, plus two more steps' worth for the epilogue.  A dropped or
  duplicated product |a w| is S / K on average: at K = 64 that is ~500x the bound, at K = 4096 still ~4x.
- act: quick-GELU is x * (0.5 tanh(0.851 x) + 0.5) with tanh.approx.f32, whose error the PTX ISA bounds by
  2^-10.987 (|tanh| <= 1, so this holds as an absolute bound), hence 0.5 * 2^-10.9 * |x|.  erf-GELU uses erff
  (2 ulp): 2^-21 |x|.  Both activations have slope <= 1.13, hence the 1.2 on acc.
- 2^-22 (|x| + |R|): the fp32 bias add, activation products and residual add, each rounded once.

Every assertion below that says "bit-identical" is exact (torch.equal), not a tolerance.
"""
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

FLAVOURS = [(act, res) for res in (False, True) for act in (0, 1, 2)]   # compile-time SPEC = act | res << 2


def _sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def pick_bn(M, N, sms):
    """gemm.cu gemm_pick_bn, recomputed: 128-wide column blocks unless the grid would under-fill the device."""
    mb = (M + 127) // 128
    if mb * ((N + 127) // 128) < sms and N >= 64:
        return 32 if mb * ((N + 63) // 64) < sms else 64
    return 128


def gemm(A, W, out, bias=None, residual=None, res_ld=0, res_row_mod=0, res_row_off=0, out_ld=0, out_group=0, act=0,
         ln_stats=None, ln_c=None, ln_w=0, stats_out=None, bn=0, generic=False, M=None):
    """b200_gemm_bf16_ex_device; returns the C status (the caller checks it)."""
    import torch
    from clip_retrieval_b200._lib import lib, GemmEpilogueC

    p = lambda t: t.data_ptr() if t is not None else None   # noqa: E731
    ep = GemmEpilogueC(p(bias), p(residual), res_ld, res_row_mod, res_row_off, out_ld, out_group, act,
                       p(ln_stats), p(ln_c), ln_w, p(stats_out))
    M = A.shape[0] if M is None else M
    return lib.b200_gemm_bf16_ex_device(A.data_ptr(), W.data_ptr(), out.data_ptr(), M, W.shape[0], A.shape[1], ep, bn,
                                        int(generic), 0, torch.cuda.current_stream().cuda_stream)


def run(*args, **kw):
    import torch
    from clip_retrieval_b200._lib import check

    check(gemm(*args, **kw), "gemm")
    torch.cuda.synchronize()


def operands(M, N, K, seed, a_scale=0.5, w_scale=0.05):
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    A = (torch.randn(M, K, device="cuda", generator=g) * a_scale).bfloat16()
    W = (torch.randn(N, K, device="cuda", generator=g) * w_scale).bfloat16()
    b = torch.randn(N, device="cuda", generator=g)
    R = torch.randn(M, N, device="cuda", generator=g).bfloat16()
    return A, W, b, R


def product64(A, W, bias):
    """(x, S): A.W^T (+ bias) and |A|.|W|^T in float64."""
    A64, W64 = A.double(), W.double()
    x = A64 @ W64.t()
    if bias is not None:
        x = x + bias.double()
    return x, A64.abs() @ W64.abs().t()


def epilogue64(x, S, K, act, R):
    """(y, bound) of the module docstring."""
    import torch

    acc = (math.ceil(K / 16) + 2) * 2.0 ** -22 * S
    if act == 1:
        y = x * torch.sigmoid(1.702 * x)
        e = 1.2 * acc + 0.5 * 2.0 ** -10.9 * x.abs()
    elif act == 2:
        y = 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))
        e = 1.2 * acc + 2.0 ** -21 * x.abs()
    else:
        y, e = x, acc.clone()
    e = e + 2.0 ** -22 * x.abs()
    if R is not None:
        R64 = R.double()
        y = y + R64
        e = e + 2.0 ** -22 * R64.abs()
    return y, 2.0 ** -8 * (y.abs() + e) + e


def assert_close(out, y, bound, what=""):
    import torch

    got = out.double()
    assert not torch.isnan(got).any(), "%s: NaN in the output" % what
    err = (got - y).abs()
    bad = err > bound
    if bool(bad.any()):
        i = int(torch.nonzero(bad.flatten())[0])
        pytest.fail("%s: %d elements out of bound; first at flat index %d: got %r ref %r bound %r (max err/bound %g)"
                    % (what, int(bad.sum()), i, got.flatten()[i].item(), y.flatten()[i].item(),
                       bound.flatten()[i].item(), (err / bound).max().item()))


# ---- the stand-alone entry (gemm_pick_bn's width, compile-time flavours) ---------------------------------------

@pytest.mark.timeout(120)
@pytest.mark.parametrize(
    "M,N,K,act,bias,res",
    [
        (128, 256, 64, 0, False, False),
        (1, 512, 512, 0, True, False),        # single row (B=1 serving shape)
        (257, 768, 768, 1, True, True),       # ragged M
        (77 * 3, 2304, 768, 0, True, False),  # text QKV
        (1000, 3072, 1024, 2, True, True),
        (300, 1280, 1280, 0, True, True),     # H/14 width, 32-wide column blocks (30 tiles of 128 would under-fill)
        (130, 520, 328, 1, True, True),       # N, K not multiples of the tile: TMA zero fill + predication
        (4112, 4096, 1024, 1, True, False),
        (4112, 1024, 4096, 0, True, True),
        (20001, 3072, 1024, 1, True, True),   # full grid, ragged M
        (19000, 1000, 520, 2, True, True),    # full grid, N and K tails
    ],
)
def test_gemm_matches_fp32_reference(M, N, K, act, bias, res):
    """The stand-alone entry against the float64 reference; its automatic column-block width is the one
    gemm_pick_bn computes from the device's SM count (the same bits as that width forced)."""
    import torch
    from clip_retrieval_b200._lib import lib, check

    A, W, b, R = operands(M, N, K, M + 31 * N + 977 * K)
    b = b if bias else None
    R = R if res else None
    out = torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
    st = torch.cuda.current_stream().cuda_stream
    check(lib.b200_gemm_bf16_device(A.data_ptr(), W.data_ptr(), b.data_ptr() if bias else None,
                                    R.data_ptr() if res else None, out.data_ptr(), M, N, K, act, 0, st), "gemm")
    torch.cuda.synchronize()
    x, S = product64(A, W, b)
    y, bound = epilogue64(x, S, K, act, R)
    assert_close(out, y, bound, "M=%d N=%d K=%d" % (M, N, K))
    forced = torch.full_like(out, float("nan"))
    run(A, W, forced, bias=b, residual=R, act=act, bn=pick_bn(M, N, _sms()))
    assert torch.equal(out, forced), "automatic width differs from gemm_pick_bn's width forced"


@pytest.mark.timeout(300)
@pytest.mark.parametrize("M,N,K,act,bias,res", [
    (20001, 3072, 1024, 1, True, False),   # qkv / fc shape class, ragged M
    (20001, 1024, 1024, 0, True, True),    # out-proj: residual stored in place of it
    (19000, 1000, 520, 2, True, True),     # N and K tails: boxes clipped by the tensor maps
    (40000, 768, 3072, 0, True, True),     # text c_proj shape class
    (20001, 512, 1024, 0, True, False),    # plain bias epilogue (qkv)
    (20001, 1024, 1024, 1, True, True),    # QuickGELU + residual
    (20001, 1024, 512, 2, False, False),   # erf-GELU, no bias
])
def test_pair_gemm_tma_store_equals_register_store(M, N, K, act, bias, res):
    """Full-grid shapes (128-wide column blocks, many waves) with every epilogue flavour: the result stored into a
    fresh buffer and the result stored over its own residual (in-place update of the residual stream, as the model
    runs it) are bit-identical, and both are within the float64 bound."""
    import torch
    from clip_retrieval_b200._lib import lib, check

    A, W, b, R = operands(M, N, K, M + 31 * N + 977 * K)
    b = b if bias else None
    R = R if res else None
    st = torch.cuda.current_stream().cuda_stream
    outs = []
    for in_place in (False, True):
        out = R.clone() if (res and in_place) else torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
        check(lib.b200_gemm_bf16_device(A.data_ptr(), W.data_ptr(), b.data_ptr() if bias else None,
                                        (out if in_place else R).data_ptr() if res else None, out.data_ptr(), M, N, K, act, 0,
                                        st), "gemm")
        torch.cuda.synchronize()
        outs.append(out)
    assert torch.equal(outs[0], outs[1]), "in-place vs separate output: max diff %g" % (outs[0].float() - outs[1].float()).abs().max().item()
    x, S = product64(A, W, b)
    y, bound = epilogue64(x, S, K, act, R)
    assert_close(outs[0], y, bound, "M=%d N=%d K=%d" % (M, N, K))


# ---- every tile width x every epilogue flavour at the tile edges -------------------------------------------------

EDGE_SHAPES = [
    (1, 8, 8),          # one row, one 8-column group, K far below one 64-column block
    (64, 40, 72),       # N tail inside every width; K one block + 8
    (65, 72, 328),      # M one past a warpgroup's 64 rows; K tail of 8 after 5 blocks
    (127, 520, 40),     # K below one block; N = 4 x 128 + 8
    (128, 136, 1024),   # exactly one row block; 16 k-blocks wrap the 3- and 4-stage rings 4-5 times
    (129, 200, 136),    # one row past a row block
    (257, 520, 4104),   # 65 k-blocks, K tail
    (2177, 264, 200),   # 18 row blocks: past the 16-row-block raster group, all column blocks
]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("bn", [32, 64, 128])
@pytest.mark.parametrize("M,N,K", EDGE_SHAPES)
def test_every_width_and_flavour_matches_float64(M, N, K, bn):
    """Each compile-time epilogue flavour (activation none / quick-GELU / erf-GELU, with and without residual) at a
    forced column-block width: within the float64 bound, bit-identical to the run-time flavour (SPEC = -1) on the
    same inputs, and, with a residual, bit-identical when the residual is the output itself (in-place update)."""
    import torch

    A, W, b, R = operands(M, N, K, M + 31 * N + 977 * K)
    x, S = product64(A, W, b)
    for act, res in FLAVOURS:
        what = "bn=%d act=%d res=%d" % (bn, act, res)
        Rr = R if res else None
        outs = []
        for generic in (False, True):
            out = torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
            run(A, W, out, bias=b, residual=Rr, act=act, bn=bn, generic=generic)
            outs.append(out)
        y, bound = epilogue64(x, S, K, act, Rr)
        assert_close(outs[0], y, bound, what)
        assert torch.equal(outs[0], outs[1]), "%s: run-time flavour differs from the compile-time flavour" % what
        if res:
            inplace = R.clone()
            run(A, W, inplace, bias=b, residual=inplace, act=act, bn=bn)
            assert torch.equal(inplace, outs[0]), "%s: in-place residual differs from a separate one" % what


@pytest.mark.timeout(300)
@pytest.mark.parametrize("M,N,K,act", [(1, 520, 328, 1), (129, 200, 1024, 0), (257, 1024, 1024, 2), (2177, 264, 200, 1)])
def test_widths_are_bit_identical_to_each_other(M, N, K, act):
    """The column-block width changes which CTA computes an element, not how: every element is the same k16 wgmma
    sequence over the same k-blocks whatever the width, so 32-, 64- and 128-wide tiles store the same bits."""
    import torch

    A, W, b, R = operands(M, N, K, 5 + M + N + K)
    outs = {}
    for bn in (32, 64, 128):
        outs[bn] = torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
        run(A, W, outs[bn], bias=b, residual=R, act=act, bn=bn)
    assert torch.equal(outs[32], outs[64]) and torch.equal(outs[64], outs[128])


@pytest.mark.timeout(120)
@pytest.mark.parametrize("bn", [32, 64, 128])
@pytest.mark.parametrize("M,N,K", [(65, 40, 72), (300, 520, 200), (129, 8, 64)])
def test_nothing_is_written_outside_the_output(M, N, K, bn):
    """Output of leading dimension N + 24 and 3 rows past M, pre-filled with NaN: columns >= N of every row and rows
    >= M stay NaN (a tile that reaches past N or M is predicated, not clipped by the allocation)."""
    import torch

    A, W, b, R = operands(M, N, K, 17 * M + N + K)
    ld = N + 24
    buf = torch.full((M + 3, ld), float("nan"), device="cuda", dtype=torch.bfloat16)
    for act, res in FLAVOURS:
        buf.fill_(float("nan"))
        Rp = torch.zeros(M, ld, device="cuda", dtype=torch.bfloat16)
        Rp[:, :N] = R
        run(A, W, buf, bias=b, residual=Rp if res else None, res_ld=ld, out_ld=ld, act=act, bn=bn)
        x, S = product64(A, W, b)
        y, bound = epilogue64(x, S, K, act, R if res else None)
        assert_close(buf[:M, :N], y, bound, "bn=%d act=%d res=%d" % (bn, act, res))
        assert bool(torch.isnan(buf[:M, N:].float()).all()), "columns past N were written"
        assert bool(torch.isnan(buf[M:].float()).all()), "rows past M were written"


@pytest.mark.timeout(120)
@pytest.mark.parametrize("grid,width,patch,B", [(7, 768, 32, 3), (16, 1024, 14, 2)])
@pytest.mark.parametrize("bn", [0, 32, 64, 128])
def test_patch_embedding_epilogue_skips_cls_rows(grid, width, patch, B, bn):
    """The patch-embedding GEMM (ViT-B/32 and ViT-L/14 grids): product row r = b * g^2 + p goes to output row
    b * (g^2 + 1) + 1 + p and adds positional row 1 + p.  The cls rows (b * (g^2 + 1)) are never written."""
    import torch

    gg = grid * grid
    K = (3 * patch * patch + 63) // 64 * 64
    M = B * gg
    A, W, b, _ = operands(M, width, K, grid + width + bn)
    g = torch.Generator(device="cuda").manual_seed(3)
    pos = torch.randn(gg + 1, width, device="cuda", generator=g).bfloat16()
    out = torch.full((B * (gg + 1), width), float("nan"), device="cuda", dtype=torch.bfloat16)
    run(A, W, out, residual=pos, res_row_mod=gg, res_row_off=1, out_group=gg, bn=bn)
    x, S = product64(A, W, None)
    idx = torch.arange(M, device="cuda")
    y, bound = epilogue64(x, S, K, 0, pos[1 + idx % gg])
    o = out.view(B, gg + 1, width)
    assert bool(torch.isnan(o[:, 0].float()).all()), "a cls row was written"
    assert_close(o[:, 1:].reshape(M, width), y, bound, "patch rows")


# ---- the model's layer shapes at serving batches --------------------------------------------------------------

def _layer_cases():
    """(arch, tower, batch): vision towers of ViT-B/32, ViT-L/14, ViT-H/14 (width 1280) and the text towers of
    ViT-B/32 and ViT-L/14, at batches 1, 2 and 8."""
    out = []
    for arch, tower in (("ViT-B/32", "vision"), ("ViT-B/32", "text"), ("ViT-L/14", "vision"), ("ViT-L/14", "text"),
                        ("ViT-H/14", "vision")):
        for B in (1, 2, 8):
            out.append((arch, tower, B))
    return out


@pytest.mark.timeout(300)
@pytest.mark.parametrize("arch,tower,B", _layer_cases())
def test_model_layer_shapes_match_float64(arch, tower, B):
    """qkv, out-proj (+ residual in place), fc (+ activation) and c_proj (+ residual in place) of one block at the
    widths the model picks: float64 bound, and the automatic width equals gemm_pick_bn's width forced."""
    import torch
    import clip_retrieval_b200 as m

    a = m.ARCHS[arch]
    t = getattr(a, tower)
    T = (a.image_size // a.patch) ** 2 + 1 if tower == "vision" else a.context_length
    M, w = B * T, t.width
    act = 1 if a.quick_gelu else 2
    sms = _sms()
    for name, N, K, act_, res in (("qkv", 3 * w, w, 0, False), ("out", w, w, 0, True), ("fc", t.mlp, w, act, False),
                                  ("proj", w, t.mlp, 0, True)):
        A, W, b, R = operands(M, N, K, M * 7 + N + K, w_scale=K ** -0.5)
        Rr = R if res else None
        auto = R.clone() if res else torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
        run(A, W, auto, bias=b, residual=auto if res else None, act=act_)
        x, S = product64(A, W, b)
        y, bound = epilogue64(x, S, K, act_, Rr)
        assert_close(auto, y, bound, "%s %s B=%d %s" % (arch, tower, B, name))
        bn = pick_bn(M, N, sms)
        forced = torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
        run(A, W, forced, bias=b, residual=Rr, act=act_, bn=bn)
        assert torch.equal(auto, forced), "%s: automatic width differs from the forced width %d" % (name, bn)


# ---- row statistics and the folded LayerNorm (the run-time flavour's own features) ------------------------------

def slotted_rows(M, w, offset, seed):
    """Rows z + mu_r + m_{r,s}: unit-variance noise, a per-row offset of `offset` standard deviations (random sign)
    and a different mean for every 64-column slot, so that the between-slot term of a combination matters."""
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    z = torch.randn(M, w, device="cuda", generator=g)
    mu = offset * torch.sign(torch.randn(M, 1, device="cuda", generator=g))
    ms = (torch.randn(M, w // 64, 1, device="cuda", generator=g) * 0.75).expand(M, w // 64, 64).reshape(M, w)
    return z + mu + ms


def slot_stats64(x):
    """float64 (mean, M2) of every 64-column slot of x: [M, w / 64, 2]."""
    v = x.double().view(x.shape[0], -1, 64)
    mean = v.mean(-1)
    return mean, ((v - mean[..., None]) ** 2).sum(-1), (v - mean[..., None]).abs().amax(-1)


def assert_records(rec, x, what):
    """fp32 shifted / two-pass sums of 64 values: |mean err| <= 2^-18 (|mean| + r), |M2 err| <= 2^-16 * 64 r^2 with r
    the slot's largest |x - mean| (the shift is within 2r of every value)."""
    mean, m2, r = slot_stats64(x)
    rec = rec.view(x.shape[0], -1, 2).double()
    em = (rec[..., 0] - mean).abs()
    e2 = (rec[..., 1] - m2).abs()
    assert bool((em <= 2.0 ** -18 * (mean.abs() + r)).all()), "%s: mean err %g" % (what, em.max().item())
    assert bool((e2 <= 2.0 ** -16 * 64 * r * r).all()), "%s: M2 err %g (M2 %g)" % (what, e2.max().item(), m2.max().item())


@pytest.mark.timeout(120)
@pytest.mark.parametrize("w", [64, 768, 1536])
@pytest.mark.parametrize("offset", [0, 8, 64])
def test_row_stats_records_match_float64(w, offset):
    import torch
    from clip_retrieval_b200._lib import lib, check

    M = 333
    x = slotted_rows(M, w, offset, w + offset).bfloat16()
    rec = torch.full((M, w // 64, 2), float("nan"), device="cuda")
    check(lib.b200_row_stats_bf16_device(x.data_ptr(), M, w, rec.data_ptr(), 0,
                                         torch.cuda.current_stream().cuda_stream), "row_stats")
    torch.cuda.synchronize()
    assert_records(rec, x, "row_stats w=%d offset=%d" % (w, offset))


@pytest.mark.timeout(120)
@pytest.mark.parametrize("M,N,K", [(1, 768, 768), (300, 1024, 4096), (257, 1536, 200), (2177, 128, 64)])
@pytest.mark.parametrize("offset", [0, 64])
def test_residual_gemm_row_statistics_match_float64(M, N, K, offset):
    """stats_out of a residual GEMM (what the out-proj / c_proj GEMMs write for the next folded LayerNorm), taken of
    the bf16 values actually stored, at the automatic width and forced to 128; the stored values are the same bits
    as without statistics."""
    import torch

    A, W, b, _ = operands(M, N, K, M + N + K + offset, w_scale=K ** -0.5)
    R = slotted_rows(M, N, offset, M + N).bfloat16()
    ref = R.clone()
    run(A, W, ref, bias=b, residual=ref)
    for bn in (0, 128):
        out = R.clone()
        rec = torch.full((M, N // 64, 2), float("nan"), device="cuda")
        run(A, W, out, bias=b, residual=out, stats_out=rec, bn=bn)
        assert torch.equal(out, ref), "row statistics changed the stored values"
        assert_records(rec, out, "stats_out M=%d N=%d bn=%d" % (M, N, bn))


@pytest.mark.timeout(60)
def test_invalid_epilogues_are_refused():
    import torch
    from clip_retrieval_b200._lib import B200Error

    A, W, b, R = operands(128, 256, 64, 1)
    out = torch.empty(128, 256, device="cuda", dtype=torch.bfloat16)
    rec = torch.empty(128, 4, 2, device="cuda")
    c = torch.zeros(256, device="cuda")
    for bn in (32, 64):
        assert gemm(A, W, out, stats_out=rec, bn=bn) == -1                       # B200_ERR_INVALID
    assert gemm(A, W, out, bn=96) == -1
    assert gemm(A, W, out, act=3) == -1
    big = torch.zeros(128, 1600 // 64, 2, device="cuda")
    assert gemm(A, W, out, ln_stats=big, ln_c=c, ln_w=1600) == -5               # B200_ERR_UNSUPPORTED
    assert gemm(A, W, out, ln_stats=big, ln_c=c, ln_w=100) == -1
    assert gemm(A, W, out, ln_stats=big, ln_w=64) == -1
    with pytest.raises(B200Error):
        run(A, W, out, stats_out=rec, bn=64)


def fold_operands(N, w, seed):
    """W [N, w], gamma, beta, bias; W' = bf16(W * gamma), c = sum_k W', d = W . beta + bias (as clip_model.cu folds)."""
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    W = (torch.randn(N, w, device="cuda", generator=g) * w ** -0.5).bfloat16()
    gamma = 1 + 0.3 * torch.randn(w, device="cuda", generator=g)
    beta = 0.2 * torch.randn(w, device="cuda", generator=g)
    bias = 0.1 * torch.randn(N, device="cuda", generator=g)
    Wp = (W.double() * gamma.double()).bfloat16()
    c = Wp.double().sum(1).float()
    d = (W.double() @ beta.double() + bias.double()).float()
    return W, gamma, beta, bias, Wp, c, d


def fold_reference(x, Wp, c, d):
    """(pre, e): the fold's contract rstd * (x W'^T - mean * c) + d with mean / rstd in float64 (eps 1e-5), and its
    error bound before the activation and the bf16 store.  Beyond the GEMM's own accumulation term (on
    S = |x| . |W'|^T, scaled by rstd): the fp32 records and their combination (mean and rstd each to 2^-19
    relative), and the two fp32 fused multiply-adds of the epilogue."""
    import torch

    x64, W64 = x.double(), Wp.double()
    w = x.shape[1]
    mean = x64.mean(1, keepdim=True)
    rstd = 1 / torch.sqrt(((x64 - mean) ** 2).sum(1, keepdim=True) / w + 1e-5)
    sig = 1 / rstd
    p = x64 @ W64.t()
    core = rstd * (p - mean * c.double())
    pre = core + d.double()
    S = x64.abs() @ W64.abs().t()
    acc = rstd * (math.ceil(w / 16) + 2) * 2.0 ** -22 * S
    e = acc + 2.0 ** -19 * (core.abs() + rstd * c.double().abs() * (mean.abs() + sig)) + 2.0 ** -22 * (
        rstd * p.abs() + rstd * (mean * c.double()).abs() + d.double().abs())
    return pre, e


def fold_bound(pre, e, act):
    """(y, bound) after the activation (0 or quick-GELU) and the bf16 store, as in epilogue64."""
    import torch

    if act == 1:
        y = pre * torch.sigmoid(1.702 * pre)
        e = 1.2 * e + 0.5 * 2.0 ** -10.9 * pre.abs()
    else:
        y = pre
    e = e + 2.0 ** -22 * pre.abs()
    return y, 2.0 ** -8 * (y.abs() + e) + e


@pytest.mark.timeout(300)
@pytest.mark.parametrize("w,N,M", [(64, 192, 129), (768, 2304, 100), (1536, 1024, 257)])
@pytest.mark.parametrize("offset", [0, 8, 64])
@pytest.mark.parametrize("source", ["row_stats", "stats_out"])
def test_folded_layernorm_matches_its_contract(w, N, M, offset, source):
    """LayerNorm folded into the GEMM (gemm.cuh GemmEpilogue::ln_stats): the output is rstd * (x W'^T - mean * c) + d
    with mean and rstd of each row in float64, for records written by row_stats (the first block) and by a
    preceding residual GEMM's stats_out (every later block), at row widths 64 and 1536 (the limit) and per-row
    offsets of 0, 8 and 64 standard deviations; with and without the activation, at every width."""
    import torch
    from clip_retrieval_b200._lib import lib, check

    st = torch.cuda.current_stream().cuda_stream
    _, _, _, _, Wp, c, d = fold_operands(N, w, w + N)
    rec = torch.full((M, w // 64, 2), float("nan"), device="cuda")
    x = slotted_rows(M, w, offset, M + w + offset).bfloat16()
    if source == "row_stats":
        check(lib.b200_row_stats_bf16_device(x.data_ptr(), M, w, rec.data_ptr(), 0, st), "row_stats")
    else:
        # x += A0 W0^T + b0 in place, as the out-proj / c_proj GEMMs update the residual stream
        A0, W0, b0, _ = operands(M, w, 256, M + w, w_scale=1 / 16)
        run(A0, W0, x, bias=b0, residual=x, stats_out=rec)
    torch.cuda.synchronize()
    pre, e = fold_reference(x, Wp, c, d)
    for act in (0, 1):
        y, bound = fold_bound(pre, e, act)
        for bn in (32, 64, 128):
            out = torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
            run(x, Wp, out, bias=d, ln_stats=rec, ln_c=c, ln_w=w, act=act, bn=bn)
            assert_close(out, y, bound, "w=%d offset=%d act=%d bn=%d" % (w, offset, act, bn))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("offset", [0, 8, 64])
def test_folded_layernorm_error_against_the_unfused_path(offset):
    """Both ways to compute LayerNorm(x) W^T + b against the float64 result of exactly that: the LayerNorm kernel
    followed by the plain GEMM, and the fold.  The fold subtracts mean * c after the fp32 sum, so a row offset
    cancels there; its error must stay within twice the unfused path's (measured on H100 SXM: see DESIGN.md §4)."""
    import torch
    from clip_retrieval_b200._lib import lib, check

    st = torch.cuda.current_stream().cuda_stream
    M, w, N = 514, 1024, 3072
    W, gamma, beta, bias, Wp, c, d = fold_operands(N, w, 11)
    x = slotted_rows(M, w, offset, 12).bfloat16()
    x64 = x.double()
    ln = torch.nn.functional.layer_norm(x64, (w,), gamma.double(), beta.double(), 1e-5)
    y = ln @ W.double().t() + bias.double()
    h = torch.empty_like(x)
    check(lib.b200_layernorm_bf16_device(x.data_ptr(), h.data_ptr(), gamma.data_ptr(), beta.data_ptr(), M, w, 0, st),
          "ln")
    unfused = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    run(h, W, unfused, bias=bias)
    rec = torch.empty(M, w // 64, 2, device="cuda")
    check(lib.b200_row_stats_bf16_device(x.data_ptr(), M, w, rec.data_ptr(), 0, st), "row_stats")
    fused = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    run(x, Wp, fused, bias=d, ln_stats=rec, ln_c=c, ln_w=w)
    e_un = (unfused.double() - y).abs()
    e_fo = (fused.double() - y).abs()
    rms = lambda t: t.pow(2).mean().sqrt().item()   # noqa: E731
    print("offset %d: unfused max %.3g rms %.3g | fold max %.3g rms %.3g"
          % (offset, e_un.max().item(), rms(e_un), e_fo.max().item(), rms(e_fo)))
    assert e_fo.max().item() <= 2 * e_un.max().item() and rms(e_fo) <= 2 * rms(e_un)


@pytest.mark.timeout(300)
def test_run_time_epilogue_with_folded_layernorm_matches_oracle():
    """The run-time epilogue flavour (every feature decided per launch: LayerNorm folded into the qkv / fc GEMMs, row
    statistics written by the residual GEMMs), reached through B200_FUSE_LN=1: ViT-B/32 embeddings against the
    fp32 oracle and against the default path (separate LayerNorm kernel, compile-time epilogue flavours)."""
    import os

    import clip_retrieval_b200 as m
    from oracle import clip_ref

    cfg = clip_ref.CONFIGS["ViT-B/32"]
    sd = clip_ref.make_state_dict(cfg, seed=0)
    arch = m.ClipArch(cfg.embed_dim, cfg.image_size, cfg.patch,
                      m.Tower(cfg.vision.width, cfg.vision.layers, cfg.vision.heads, cfg.vision.mlp),
                      m.Tower(cfg.text.width, cfg.text.layers, cfg.text.heads, cfg.text.mlp),
                      cfg.context_length, cfg.vocab_size, cfg.quick_gelu)
    px, tk = clip_ref.synth_images(6, cfg, seed=4), clip_ref.synth_tokens(6, cfg, seed=4)
    outs = {}
    old = os.environ.get("B200_FUSE_LN")
    try:
        for fuse in ("0", "1"):
            os.environ["B200_FUSE_LN"] = fuse
            model = m.B200Clip(arch, device=0, max_batch=8).load_state_dict(sd)
            outs[fuse] = (model.embed_image(px), model.embed_text(tk))
            del model
    finally:
        if old is None:
            os.environ.pop("B200_FUSE_LN", None)
        else:
            os.environ["B200_FUSE_LN"] = old
    ref_i, ref_t = clip_ref.mapper_image(sd, cfg, px), clip_ref.mapper_text(sd, cfg, tk)
    for (ei, et) in outs.values():
        assert np.isfinite(ei.astype(np.float32)).all() and np.isfinite(et.astype(np.float32)).all()
        assert (1 - clip_ref.cosine(ei, ref_i)).max() <= 1e-3 and (1 - clip_ref.cosine(et, ref_t)).max() <= 1e-3
    assert (1 - clip_ref.cosine(outs["1"][0], outs["0"][0])).max() <= 1e-3
    assert (1 - clip_ref.cosine(outs["1"][1], outs["0"][1])).max() <= 1e-3


def test_model_layer_shapes_reach_every_width():
    """The model-shape cases above launch all three column-block widths on this device, 64 included (ViT-L/14
    vision qkv / fc at batch 1 and 2, for one)."""
    import clip_retrieval_b200 as m

    sms, picked = _sms(), set()
    for arch, tower, B in _layer_cases():
        a = m.ARCHS[arch]
        t = getattr(a, tower)
        T = (a.image_size // a.patch) ** 2 + 1 if tower == "vision" else a.context_length
        for N in (3 * t.width, t.width, t.mlp):
            picked.add(pick_bn(B * T, N, sms))
    assert picked == {32, 64, 128}, picked
