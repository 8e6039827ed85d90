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
         bn=0, flags=0, M=None, reserved=None):
    """b200_gemm_bf16_ex_device; returns the C status (the caller checks it).  reserved: {member: value} set in the
    epilogue struct's reserved members (which must be zero)."""
    import torch
    from clip_retrieval_b200._lib import lib, GemmEpilogueC

    p = lambda t: t.data_ptr() if t is not None else None   # noqa: E731
    ep = GemmEpilogueC(p(bias), p(residual), res_ld, res_row_mod, res_row_off, out_ld, out_group, act)
    for name, value in (reserved or {}).items():
        setattr(ep, name, value)
    M = A.shape[0] if M is None else M
    return lib.b200_gemm_bf16_ex_device(A.data_ptr(), W.data_ptr(), out.data_ptr(), M, W.shape[0], A.shape[1], ep, bn,
                                        flags, 0, torch.cuda.current_stream().cuda_stream)


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
def test_every_width_and_epilogue_matches_float64(M, N, K, bn):
    """Each epilogue flavour (activation none / quick-GELU / erf-GELU, with and without residual) at a forced
    column-block width: within the float64 bound, and, with a residual, bit-identical when the residual is the output
    itself (in-place update)."""
    import torch

    A, W, b, R = operands(M, N, K, M + 31 * N + 977 * K)
    x, S = product64(A, W, b)
    for act, res in FLAVOURS:
        what = "bn=%d act=%d res=%d" % (bn, act, res)
        Rr = R if res else None
        out = torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
        run(A, W, out, bias=b, residual=Rr, act=act, bn=bn)
        y, bound = epilogue64(x, S, K, act, Rr)
        assert_close(out, y, bound, what)
        if res:
            inplace = R.clone()
            run(A, W, inplace, bias=b, residual=inplace, act=act, bn=bn)
            assert torch.equal(inplace, out), "%s: in-place residual differs from a separate one" % what


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


@pytest.mark.timeout(60)
def test_invalid_epilogues_and_flags_are_refused():
    """B200_ERR_INVALID (-1) for an unsupported width or activation, an undefined flags bit, and a non-zero reserved
    member of the epilogue struct (the removed LayerNorm fold's inputs are refused, not ignored)."""
    import torch
    from clip_retrieval_b200._lib import B200Error

    A, W, b, R = operands(128, 256, 64, 1)
    out = torch.empty(128, 256, device="cuda", dtype=torch.bfloat16)
    assert gemm(A, W, out, bn=96) == -1
    assert gemm(A, W, out, act=3) == -1
    for bn in (0, 32, 64, 128, 256):
        assert gemm(A, W, out, bn=bn, flags=1) == -1                            # flags bit 0 is not defined
    for name, value in (("reserved0", b.data_ptr()), ("reserved1", b.data_ptr()), ("reserved2", 64),
                        ("reserved3", out.data_ptr())):
        for bn in (0, 32, 128):
            assert gemm(A, W, out, bias=b, bn=bn, reserved={name: value}) == -1, (name, bn)
    assert gemm(A, W, out, bias=b) == 0
    with pytest.raises(B200Error):
        run(A, W, out, act=3)


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
