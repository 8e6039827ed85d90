"""The TMA-store epilogue of the persistent 128 x 256 GEMM (gemm.cuh gemm_bf16_wgmma_persistent_kernel, bn = 256): the
output stored by TMA from a swizzled bf16 staging tile, the residual loaded into that tile by TMA while the k-loop runs,
and the register-store branch the row maps keep.  Every check compares against bn = 128 bit for bit (torch.equal).
"""
import pytest

from test_gemm_gpu import FLAVOURS, _sms, operands, run

pytestmark = pytest.mark.gpu

TMA = 2   # flags == 2: the TMA-store epilogue at any grid size (the library takes it from 8 tiles per SM up)


def _nan(rows, cols):
    import torch

    return torch.full((rows, cols), float("nan"), device="cuda", dtype=torch.bfloat16)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("M", [1, 65, 127, 129, 2177])
@pytest.mark.parametrize("N", [8, 40, 264, 520])
def test_strided_output_guards_stay_nan(M, N):
    """Output of leading dimension N + 40 inside a NaN-filled buffer with 5 rows past M: the tensor map clips the
    stores at M and N, so [:M, :N] matches bn = 128 and every other element is still NaN."""
    import torch

    K = 136
    A, W, b, R = operands(M, N, K, 3 * M + 7 * N)
    ld = N + 40
    for act, res in FLAVOURS:
        buf = _nan(M + 5, ld)
        run(A, W, buf, bias=b, residual=R if res else None, out_ld=ld, act=act, bn=256, flags=TMA)
        ref = _nan(M, N)
        run(A, W, ref, bias=b, residual=R if res else None, act=act, bn=128)
        what = "M=%d N=%d act=%d res=%d" % (M, N, act, res)
        assert torch.equal(buf[:M, :N], ref), "%s: differs from bn=128" % what
        assert bool(torch.isnan(buf[:M, N:].float()).all()), "%s: columns past N were written" % what
        assert bool(torch.isnan(buf[M:].float()).all()), "%s: rows past M were written" % what


@pytest.mark.timeout(120)
@pytest.mark.parametrize("M,N,K", [(65, 40, 72), (2177, 520, 200), (300, 264, 4104)])
def test_residual_ld_differs_from_output_ld(M, N, K):
    """The residual map has its own leading dimension (N + 16) and the output another (N + 72)."""
    import torch

    A, W, b, R = operands(M, N, K, 11 * M + N + K)
    Rp = _nan(M, N + 16)
    Rp[:, :N] = R
    for act in (0, 1, 2):
        buf = _nan(M, N + 72)
        run(A, W, buf, bias=b, residual=Rp, res_ld=N + 16, out_ld=N + 72, act=act, bn=256, flags=TMA)
        ref = _nan(M, N)
        run(A, W, ref, bias=b, residual=R, act=act, bn=128)
        assert torch.equal(buf[:, :N], ref), "act=%d: differs from bn=128" % act
        assert bool(torch.isnan(buf[:, N:].float()).all()), "act=%d: columns past N were written" % act


@pytest.mark.timeout(300)
@pytest.mark.parametrize("extra", ["grid-1", "grid", "grid+1", "3grid+5"])
def test_in_place_residual_across_tile_rounds(extra):
    """Residual updated in place (out == residual) with grid - 1, grid, grid + 1 and 3 grid + 5 tiles of 128 x 256: a
    CTA's store of one tile drains while its next tile's residual is loaded, on neighbouring rows.  The last row block
    is ragged."""
    import torch

    grid = _sms()
    tiles = {"grid-1": grid - 1, "grid": grid, "grid+1": grid + 1, "3grid+5": 3 * grid + 5}[extra]
    K = 328
    if tiles % 2 == 0:
        N, M = 512, tiles // 2 * 128 - 37
    else:   # one column block
        N, M = 256, tiles * 128 - 37
    A, W, b, R = operands(M, N, K, tiles)
    for act in (0, 1):
        ref = _nan(M, N)
        run(A, W, ref, bias=b, residual=R, act=act, bn=128)
        inplace = R.clone()
        run(A, W, inplace, bias=b, residual=inplace, act=act, bn=256, flags=TMA)
        assert torch.equal(inplace, ref), "tiles=%d act=%d: in-place residual differs from bn=128" % (tiles, act)


@pytest.mark.timeout(120)
@pytest.mark.parametrize("rowmap", ["out_group", "res_row_mod"])
@pytest.mark.parametrize("grid,width,patch,B", [(7, 768, 32, 5), (16, 1024, 14, 3)])
def test_row_maps_take_the_register_store_branch(rowmap, grid, width, patch, B):
    """Each row map on its own (the patch embedding sets both): the output row map with a plain residual, and the
    residual row map with a plain output, at the ViT-B/32 (49-row groups, straddling tiles) and ViT-L/14 grids; the
    row maps keep the register-store epilogue even when the TMA-store epilogue is forced."""
    import torch

    gg = grid * grid
    K = (3 * patch * patch + 63) // 64 * 64
    M = B * gg
    A, W, b, R = operands(M, width, K, grid + width)
    g = torch.Generator(device="cuda").manual_seed(5)
    pos = torch.randn(gg + 1, width, device="cuda", generator=g).bfloat16()
    outs = {}
    for bn in (128, 256):
        if rowmap == "out_group":
            outs[bn] = _nan(B * (gg + 1), width)
            run(A, W, outs[bn], bias=b, residual=R, out_group=gg, act=1, bn=bn, flags=TMA if bn == 256 else 0)
        else:
            outs[bn] = _nan(M, width)
            run(A, W, outs[bn], bias=b, residual=pos, res_row_mod=gg, res_row_off=1, act=1, bn=bn, flags=TMA if bn == 256 else 0)
    if rowmap == "out_group":
        o, o128 = outs[256].view(B, gg + 1, width), outs[128].view(B, gg + 1, width)
        assert bool(torch.isnan(o[:, 0].float()).all()), "a cls row was written"
        assert torch.equal(o[:, 1:], o128[:, 1:]), "out_group: patch rows differ from bn=128"
    else:
        assert torch.equal(outs[256], outs[128]), "res_row_mod: bn=256 differs from bn=128"
