"""The stride-1 3x3 patch path of the conv kernel (tc_conv_patch_kernel: the general path's 8 x 16 or 16 x 8 tiles, one
(bh + 2) x (bw + 2) input patch per tile and K block for all nine taps) vs torch-CPU fp64, in tf32 and bf16, at the
shapes that reach what it changes: ragged tiles (H not a multiple of 16, W not a multiple of 8), a single tile, more
tiles than CTAs (the patch slots refill across tiles), N split 2 and 4, both tile shapes, the 132-channel K tail, and the
dgrad of the 132-channel concat (wgmma N = 144).  Tolerances as in test_conv_ops_gpu.py."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = {0: 2e-3, 2: 2e-5}


def opnd(x, prec):
    return (x.bfloat16() if prec == 2 else x).double()


def rel_err(a, b):
    a = a.double().cpu()
    b = b.double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def nhwc(x_chw):
    return x_chw.permute(1, 2, 0).contiguous()


# (C, out_h, out_w, rot)
CASES = [
    (128, 37, 21, 0),     # ragged bottom and right tiles
    (128, 16, 8, 0),      # exactly one tile (N split 4)
    (128, 13, 5, 0),      # one ragged tile
    (128, 80, 80, 0),     # 16 x 8 tiles, 50 of them: N split 2
    (128, 64, 64, 0),     # 16 x 8 tiles, 32 of them: N split 4
    (132, 45, 30, 4),     # K tail: 4 real channels in the last K block
    (128, 300, 200, 0),   # 475 tiles: several tiles per CTA
    (132, 130, 66, 4),
    (64, 40, 24, 0),      # one K block (tf32) / half a block (bf16)
    (132, 40, 48, 4),     # 16 x 8 tiles with the K tail
]


@pytest.mark.parametrize("prec", [0, 2])
@pytest.mark.parametrize("case", CASES)
def test_patch_fprop(case, prec):
    import dip_engine as de
    C, oh, ow, rot = case
    g = torch.Generator().manual_seed(11)
    a = torch.randn(C, oh + 2, ow + 2, generator=g)
    w = torch.randn(128, C, 3, 3, generator=g) / (C * 9) ** 0.5
    b = torch.randn(128, generator=g)
    ref = F.conv2d(torch.roll(opnd(a, prec), rot, 0)[None], opnd(w, prec), b.double())[0]
    stats = torch.zeros(256 * 16, dtype=torch.float64, device="cuda")
    d = de.op_conv_fprop(nhwc(a).cuda(), w.cuda(), b.cuda(), 3, 1, 0, 0, oh, ow, rot=rot, stats=stats, precision=prec)
    torch.cuda.synchronize()
    assert torch.isfinite(d).all()
    assert rel_err(d.permute(2, 0, 1), ref) < TOL[prec]
    st = stats.view(256, 16)[:, 0]
    s1, s2 = ref.sum((1, 2)), (ref * ref).sum((1, 2))
    assert rel_err(st[:128], s1) < 10 * TOL[prec] + 1e-6 or (st[:128].cpu() - s1).abs().max() < 1e-2
    assert rel_err(st[128:], s2) < 10 * TOL[prec]


@pytest.mark.parametrize("prec", [0, 2])
@pytest.mark.parametrize("case", CASES)
def test_patch_dgrad(case, prec):
    """input gradient over dY (h x w): dx is (h + 2) x (w + 2), the patch reads dY at offset -2 (zeros outside)"""
    import dip_engine as de
    C, h, w_, rot = case
    g = torch.Generator().manual_seed(12)
    dy = torch.randn(128, h, w_, generator=g)
    w = torch.randn(128, C, 3, 3, generator=g) / (128 * 9) ** 0.5
    ref = torch.roll(F.conv_transpose2d(opnd(dy, prec)[None], opnd(w, prec))[0], -rot, 0)
    dx = de.op_conv_dgrad(nhwc(dy).cuda(), w.cuda(), 3, h + 2, w_ + 2, rot=rot, precision=prec)
    torch.cuda.synchronize()
    assert torch.isfinite(dx).all()
    assert rel_err(dx.permute(2, 0, 1), ref) < TOL[prec]
