"""The persistent 128 x 256 GEMM (gemm.cuh gemm_bf16_wgmma_persistent_kernel, bn = 256) against the 128-wide kernel
forced through the ex entry, bit for bit, and against the float64 bound of test_gemm_gpu.py.

Every element is the same k16 wgmma sequence over the same k-blocks whatever the tile width, and the epilogue is the
same per-element fp32 arithmetic, so "bit-identical" below is exact (torch.equal), not a tolerance.
"""
import pytest

from test_gemm_gpu import FLAVOURS, _sms, assert_close, epilogue64, gemm, operands, product64, run

pytestmark = pytest.mark.gpu

WIDE_MIN_TILES_PER_SM = 1   # gemm.cu GEMM_WIDE_MIN_TILES_PER_SM


def pick_is_wide(M, N, sms):
    """gemm.cu gemm_pick_bn, recomputed for the compile-time flavours: 256 once the 256-wide grid is large enough."""
    return ((M + 127) // 128) * ((N + 255) // 256) >= WIDE_MIN_TILES_PER_SM * sms


def nan_out(M, N):
    import torch

    return torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)


def check_against_128(A, W, b, R, act, what, bound=True):
    """bn = 256 against bn = 128 (bit-identical), the float64 bound, and with a residual the in-place update."""
    import torch

    M, N, K = A.shape[0], W.shape[0], A.shape[1]
    outs = {}
    for bn in (128, 256):
        outs[bn] = nan_out(M, N)
        run(A, W, outs[bn], bias=b, residual=R, act=act, bn=bn)
    assert torch.equal(outs[256], outs[128]), "%s: bn=256 differs from bn=128" % what
    if bound:
        x, S = product64(A, W, b)
        y, bnd = epilogue64(x, S, K, act, R)
        assert_close(outs[256], y, bnd, what)
    if R is not None:
        inplace = R.clone()
        run(A, W, inplace, bias=b, residual=inplace, act=act, bn=256)
        assert torch.equal(inplace, outs[128]), "%s: in-place residual differs from a separate one" % what


# M: one row, one past a warpgroup's rows, one short of / one past a row block (the second CTA of the pair has no
# rows), an odd number of row blocks (3), past
# the 16-row-block raster group (18 blocks).  N: one 8-column group, tails inside the 256-wide tile.  K: below one
# 64-column block, a tail of 8 after 5 blocks, 65 blocks with a tail (wraps the 4-stage ring 16 times).
EDGE_SHAPES = [
    (1, 8, 40),
    (65, 264, 328),
    (127, 520, 4104),
    (129, 264, 40),
    (300, 520, 136),
    (2177, 520, 328),
    (2177, 8, 4104),
    (65, 8, 4104),
]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("M,N,K", EDGE_SHAPES)
def test_wide_every_flavour_at_the_edges(M, N, K):
    A, W, b, R = operands(M, N, K, M + 31 * N + 977 * K)
    for act, res in FLAVOURS:
        check_against_128(A, W, b, R if res else None, act, "M=%d N=%d K=%d act=%d res=%d" % (M, N, K, act, res))


def _grid_cases():
    """(M, N, K) whose 256-wide grids are smaller than, equal to, a multiple plus one of, and not a multiple of the
    persistent grid (one CTA per SM)."""
    sms = _sms()
    return [(128 * 5, 512, 256),                 # 10 tiles
            (128 * sms, 256, 256),               # exactly one tile per CTA
            (128 * (2 * sms + 1) - 3, 256, 200),  # two tiles per CTA and one more, ragged M
            (128 * (sms + 5), 768, 136)]          # 3 (sms + 5) tiles


@pytest.mark.timeout(300)
@pytest.mark.parametrize("case", range(4))
def test_wide_persistent_grid_sizes(case):
    M, N, K = _grid_cases()[case]
    A, W, b, R = operands(M, N, K, 7 * M + N + K)
    for act, res in ((1, False), (0, True)):
        check_against_128(A, W, b, R if res else None, act, "M=%d N=%d K=%d act=%d res=%d" % (M, N, K, act, res))


@pytest.mark.timeout(120)
@pytest.mark.parametrize("M,N,K", [(65, 40, 72), (300, 520, 200), (129, 8, 64), (2177, 264, 200)])
def test_wide_writes_nothing_outside_the_output(M, N, K):
    """Output of leading dimension N + 24 and 3 rows past M, pre-filled with NaN: only [:M, :N] is written."""
    import torch

    A, W, b, R = operands(M, N, K, 17 * M + N + K)
    ld = N + 24
    buf = torch.full((M + 3, ld), float("nan"), device="cuda", dtype=torch.bfloat16)
    for act, res in FLAVOURS:
        buf.fill_(float("nan"))
        Rp = torch.zeros(M, ld, device="cuda", dtype=torch.bfloat16)
        Rp[:, :N] = R
        run(A, W, buf, bias=b, residual=Rp if res else None, res_ld=ld, out_ld=ld, act=act, bn=256)
        ref = nan_out(M, N)
        run(A, W, ref, bias=b, residual=R if res else None, act=act, bn=128)
        assert torch.equal(buf[:M, :N], ref), "act=%d res=%d: differs from bn=128" % (act, res)
        assert bool(torch.isnan(buf[:M, N:].float()).all()), "columns past N were written"
        assert bool(torch.isnan(buf[M:].float()).all()), "rows past M were written"


@pytest.mark.timeout(120)
@pytest.mark.parametrize("grid,width,patch,B", [(7, 768, 32, 5), (16, 1024, 14, 3)])
def test_wide_patch_embedding_epilogue(grid, width, patch, B):
    """out_group / res_row_mod (ViT-B/32 and ViT-L/14 grids): bit-identical to bn = 128, cls rows never written."""
    import torch

    gg = grid * grid
    K = (3 * patch * patch + 63) // 64 * 64
    M = B * gg
    A, W, _, _ = operands(M, width, K, grid + width)
    g = torch.Generator(device="cuda").manual_seed(3)
    pos = torch.randn(gg + 1, width, device="cuda", generator=g).bfloat16()
    outs = {}
    for bn in (128, 256):
        outs[bn] = nan_out(B * (gg + 1), width)
        run(A, W, outs[bn], residual=pos, res_row_mod=gg, res_row_off=1, out_group=gg, bn=bn)
    o, o128 = outs[256].view(B, gg + 1, width), outs[128].view(B, gg + 1, width)
    assert bool(torch.isnan(o[:, 0].float()).all()), "a cls row was written"
    assert torch.equal(o[:, 1:], o128[:, 1:]), "patch rows differ from bn=128"
    x, S = product64(A, W, None)
    idx = torch.arange(M, device="cuda")
    y, bound = epilogue64(x, S, K, 0, pos[1 + idx % gg])
    assert_close(o[:, 1:].reshape(M, width), y, bound, "patch rows")


# (name, M, N, K, act, residual): the ViT-L/14 layer GEMMs at batch 1024, image tower (257 tokens) and text tower (77)
VITL14_SHAPES = [
    ("img qkv", 263168, 3072, 1024, 0, False), ("img out", 263168, 1024, 1024, 0, True),
    ("img fc", 263168, 4096, 1024, 1, False), ("img proj", 263168, 1024, 4096, 0, True),
    ("txt qkv", 78848, 2304, 768, 0, False), ("txt out", 78848, 768, 768, 0, True),
    ("txt fc", 78848, 3072, 768, 1, False), ("txt proj", 78848, 768, 3072, 0, True),
]


@pytest.mark.timeout(600)
@pytest.mark.parametrize("shape", VITL14_SHAPES, ids=[s[0] for s in VITL14_SHAPES])
def test_wide_vitl14_layer_shapes(shape):
    """The bench shapes: the automatic pick launches the persistent kernel (seen in a profile of the launch), bit-identical
    to bn = 128, the residual updated in place as the model runs it; 1024 rows of the result checked against the
    float64 bound."""
    import torch

    from torch.profiler import ProfilerActivity, profile

    name, M, N, K, act, res = shape
    assert pick_is_wide(M, N, _sms())
    A, W, b, R = operands(M, N, K, M + N + K, w_scale=K ** -0.5)
    R = R if res else None
    auto = R.clone() if res else nan_out(M, N)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(A, W, auto, bias=b, residual=auto if res else None, act=act)
    launched = [e.name for e in prof.events() if "gemm_bf16" in e.name]
    assert len(launched) == 1 and "persistent" in launched[0], "%s: the automatic pick launched %r" % (name, launched)
    ref = nan_out(M, N)
    run(A, W, ref, bias=b, residual=R, act=act, bn=128)
    assert torch.equal(auto, ref), "%s: automatic pick differs from bn=128" % name
    rows = torch.cat([torch.arange(512, device="cuda"), torch.arange(M - 512, M, device="cuda")])
    x, S = product64(A[rows], W, b)
    y, bound = epilogue64(x, S, K, act, R[rows] if res else None)
    assert_close(auto[rows], y, bound, name)


@pytest.mark.timeout(60)
def test_wide_refusals():
    """bn = 256 with an undefined flags bit (bit 0, alone or beside the TMA-store bit) or a non-zero reserved member
    of the epilogue struct (the removed LayerNorm fold's row statistics and inputs) is refused with B200_ERR_INVALID
    (-1); without them it runs."""
    import torch

    A, W, b, R = operands(128, 256, 64, 1)
    out = torch.empty(128, 256, device="cuda", dtype=torch.bfloat16)
    rec = torch.zeros(128, 4, 2, device="cuda")
    assert gemm(A, W, out, bias=b, bn=256, flags=1) == -1
    assert gemm(A, W, out, bias=b, residual=R, bn=256, flags=3) == -1
    assert gemm(A, W, out, bias=b, residual=R, bn=256, reserved={"reserved3": rec.data_ptr()}) == -1
    assert gemm(A, W, out, bias=b, bn=256, reserved={"reserved0": rec.data_ptr(), "reserved2": 64}) == -1
    assert gemm(A, W, out, bias=b, bn=256) == 0
    torch.cuda.synchronize()


def _auto_kernel(M, N, K, act, res):
    import torch
    from torch.profiler import ProfilerActivity, profile

    A, W, b, R = operands(M, N, K, 1)
    out = nan_out(M, N)
    run(A, W, out, bias=b, residual=R if res else None, act=act)   # warm-up outside the profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(A, W, out, bias=b, residual=R if res else None, act=act)
    names = [e.name for e in prof.events() if "gemm_bf16" in e.name]
    assert len(names) == 1, names
    return names[0]


@pytest.mark.timeout(300)
def test_automatic_pick_reaches_the_wide_kernel_at_the_bench_shapes():
    """ViT-L/14 at batch 1024 launches the persistent kernel; the ViT-H/14 text tower at batches 1 and 8 does not."""
    sms = _sms()
    for name, M, N, K, act, res in VITL14_SHAPES[4:]:
        assert "persistent" in _auto_kernel(M, N, K, act, res), name
    for B in (1, 8):
        M = 77 * B
        for N, K, act, res in ((3072, 1024, 0, False), (1024, 1024, 0, True), (4096, 1024, 2, False), (1024, 4096, 0, True)):
            assert not pick_is_wide(M, N, sms)
            assert "persistent" not in _auto_kernel(M, N, K, act, res), (B, N, K)
