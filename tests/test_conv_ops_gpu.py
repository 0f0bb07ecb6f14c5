"""P1 (kernel tier): the wgmma / SIMT convolution kernels behind the C ABI vs torch-CPU fp64 (SURVEY.md 7.4).

Tolerances: fp32 mode <= 2e-6 relative Frobenius error; tf32 mode <= 2e-3 (10-bit mantissa operands, fp32 accumulate);
bf16 mode (precision 2, wgmma bf16): the reference is evaluated on the operands ROUNDED TO BF16 (what the kernel
reads), products and sums in fp64 -> only the fp32 accumulation differs: <= 2e-5.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = {0: 2e-3, 1: 2e-6, 2: 2e-5}


def opnd(x, prec):
    """the operand as the kernel of precision mode `prec` reads it, in fp64"""
    return (x.bfloat16() if prec == 2 else x).double()


def rel_err(a, b):
    a = a.double().cpu()
    b = b.double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def nhwc(x_chw):
    return x_chw.permute(1, 2, 0).contiguous()


CASES = [
    # (C, k, stride, out_h, out_w, rot)
    (128, 1, 1, 32, 32, 0),
    (128, 3, 1, 32, 32, 0),
    (32, 3, 2, 32, 32, 0),
    (128, 3, 2, 16, 16, 0),
    (132, 3, 1, 32, 32, 4),
    (128, 3, 1, 24, 36, 0),
    (132, 3, 1, 2, 2, 4),
    (128, 3, 1, 64, 128, 0),
    (128, 3, 1, 256, 256, 0),     # >= 2 waves of tiles: persistent CTAs walk several tiles each
    (132, 3, 1, 200, 312, 4),
    (128, 1, 1, 256, 512, 0),
    (128, 3, 1, 270, 150, 0),     # several waves of tiles with ragged right / bottom tiles
]


@pytest.mark.parametrize("prec", [1, 0, 2])
@pytest.mark.parametrize("case", CASES)
def test_fprop(case, prec):
    import dip_engine as de
    C, k, stride, oh, ow, rot = case
    g = torch.Generator().manual_seed(1)
    ih, iw = (oh - 1) * stride + k, (ow - 1) * stride + k
    if stride == 2:  # engine buffers are padded to even extents
        ih += ih % 2
        iw += iw % 2
    a = torch.randn(C, ih, iw, generator=g)
    w = torch.randn(128, C, k, k, generator=g) / (C * k * k) ** 0.5
    b = torch.randn(128, generator=g)
    ref = F.conv2d(torch.roll(opnd(a, prec), rot, 0)[None], opnd(w, prec), b.double(), stride=stride)[0][:, :oh, :ow]
    stats = torch.zeros(256 * 16, dtype=torch.float64, device="cuda")   # one accumulator per 128-byte line
    d = de.op_conv_fprop(nhwc(a).cuda(), w.cuda(), b.cuda(), k, stride, 0, 0, oh, ow, rot=rot, stats=stats,
                         precision=prec)
    torch.cuda.synchronize()
    err = rel_err(d.permute(2, 0, 1), ref)
    assert err < TOL[prec], err
    s1 = ref.sum((1, 2))
    s2 = (ref * ref).sum((1, 2))
    st = stats.view(256, 16)[:, 0]
    assert rel_err(st[:128], s1) < 10 * TOL[prec] + 1e-6 or (st[:128].cpu() - s1).abs().max() < 1e-2
    assert rel_err(st[128:], s2) < 10 * TOL[prec]


@pytest.mark.parametrize("prec", [1, 0, 2])
@pytest.mark.parametrize("case", [(128, 3, 32, 32, 0), (132, 3, 32, 32, 4), (128, 1, 32, 32, 0), (128, 3, 10, 20, 0),
                                  (132, 3, 2, 2, 4), (128, 3, 64, 128, 0), (128, 3, 254, 254, 0), (132, 3, 200, 312, 4), (128, 3, 268, 148, 0)])
def test_dgrad(case, prec):
    import dip_engine as de
    C, k, h, w_, rot = case
    g = torch.Generator().manual_seed(2)
    dy = torch.randn(128, h, w_, generator=g)
    w = torch.randn(128, C, k, k, generator=g) / (128 * k * k) ** 0.5
    ref = torch.roll(F.conv_transpose2d(opnd(dy, prec)[None], opnd(w, prec))[0], -rot, 0)
    dx = de.op_conv_dgrad(nhwc(dy).cuda(), w.cuda(), k, h + k - 1, w_ + k - 1, rot=rot, precision=prec)
    torch.cuda.synchronize()
    err = rel_err(dx.permute(2, 0, 1), ref)
    assert err < TOL[prec], err


@pytest.mark.parametrize("prec", [1, 0, 2])
@pytest.mark.parametrize("case", CASES)
def test_wgrad(case, prec):
    import dip_engine as de
    C, k, stride, oh, ow, rot = case
    g = torch.Generator().manual_seed(3)
    ih, iw = (oh - 1) * stride + k, (ow - 1) * stride + k
    if stride == 2:
        ih += ih % 2
        iw += iw % 2
    a = torch.randn(C, ih, iw, generator=g)
    dy = torch.randn(128, oh, ow, generator=g)
    ia, ja = (oh - 1) * stride + k, (ow - 1) * stride + k
    ref = torch.nn.grad.conv2d_weight(torch.roll(opnd(a, prec), rot, 0)[None, :, :ia, :ja], (128, C, k, k),
                                      opnd(dy, prec)[None], stride=stride)
    dw = de.op_conv_wgrad(nhwc(dy).cuda(), nhwc(a).cuda(), C, k, stride, 0, 0, rot=rot, precision=prec)
    torch.cuda.synchronize()
    err = rel_err(dw, ref)
    assert err < TOL[prec], err


@pytest.mark.parametrize("prec", [1, 0, 2])
@pytest.mark.parametrize("case", [(128, 16, 16), (128, 64, 64), (128, 129, 128), (32, 40, 24), (128, 9, 13), (128, 2, 2)])
def test_dgrad_stride2_phases(case, prec):
    """Input gradient of the 3x3 stride-2 convs read from dY at its own resolution (tensor cores: four sub-pixel phase
    GEMMs in one launch; fp32: the SIMT kernel over dY dilated by 2), vs conv_transpose2d(stride=2) in fp64.  dx is the
    padded (2h+2) x (2w+2) gradient: the transposed conv covers (2h+1) x (2w+1), the last row / column receive no tap and
    must come out as exact zeros (never left unwritten)."""
    import dip_engine as de
    C, h, w_ = case
    g = torch.Generator().manual_seed(4)
    dy = torch.randn(128, h, w_, generator=g)
    w = torch.randn(128, C, 3, 3, generator=g) / (128 * 9) ** 0.5
    ref = F.conv_transpose2d(opnd(dy, prec)[None], opnd(w, prec), stride=2)[0]          # C x (2h+1) x (2w+1)
    dx = de.op_conv_dgrad_s2(nhwc(dy).cuda(), w.cuda(), precision=prec)
    torch.cuda.synchronize()
    assert torch.isfinite(dx).all(), "part of the padded gradient was never written"
    got = dx.permute(2, 0, 1).cpu()
    assert rel_err(got[:, :2 * h + 1, :2 * w_ + 1], ref) < TOL[prec]
    assert got[:, 2 * h + 1, :].abs().max() == 0 and got[:, :, 2 * w_ + 1].abs().max() == 0


@pytest.mark.parametrize("op", ["fprop", "dgrad", "dgrad_s2", "wgrad"])
def test_bf16_operands_too_large_for_the_scratch_are_refused(op):
    """In bf16 the single-op entry points copy their operands to bf16 inside the caller's scratch area.  A 1024 x 1024 x
    128 operand (256 MB as bf16, more than dip_op_scratch_bytes()) is refused with an error that names the scratch,
    before anything is launched: the caller's NaN-filled output is left as it was."""
    import dip_engine as de
    L = de.lib()
    h, w_ = 1024, 1024
    big = torch.zeros(h, w_, 128, device="cuda")   # NHWC: the input of the fprop, dY of the other three
    assert h * w_ * 128 * 2 > L.dip_op_scratch_bytes()
    nan = float("nan")
    scratch, s = de._ptr(de._get_scratch(big.device)), de._stream()
    if op == "fprop":
        w, b = torch.zeros(128, 128, 1, 1, device="cuda"), torch.zeros(128, device="cuda")
        out = torch.full((h, w_, 128), nan, device="cuda")
        rc = L.dip_op_conv_fprop(de._ptr(big), h, w_, 128, de._ptr(w), de._ptr(b), 128, 128, 1, 1, 0, 0, 0, de._ptr(out), h,
                                 w_, None, de.PRECISION_BF16, scratch, s)
    elif op == "dgrad":
        w = torch.zeros(128, 4, 3, 3, device="cuda")
        out = torch.full((h + 2, w_ + 2, 4), nan, device="cuda")
        rc = L.dip_op_conv_dgrad(de._ptr(big), h, w_, de._ptr(w), 128, 4, 3, 0, de._ptr(out), h + 2, w_ + 2,
                                 de.PRECISION_BF16, scratch, s)
    elif op == "dgrad_s2":
        w = torch.zeros(128, 4, 3, 3, device="cuda")
        out = torch.full((2 * h + 2, 2 * w_ + 2, 4), nan, device="cuda")
        rc = L.dip_op_conv_dgrad_s2(de._ptr(big), h, w_, de._ptr(w), 128, 4, 0, de._ptr(out), de.PRECISION_BF16, scratch, s)
    else:
        a = torch.zeros(h, w_, 4, device="cuda")
        out = torch.full((128, 4, 1, 1), nan, device="cuda")
        rc = L.dip_op_conv_wgrad(de._ptr(big), h, w_, de._ptr(a), h, w_, 4, 128, 4, 1, 1, 0, 0, 0, de._ptr(out),
                                 de.PRECISION_BF16, scratch, s)
    with pytest.raises(RuntimeError, match="scratch"):
        de.check(rc)
    torch.cuda.synchronize()
    assert torch.isnan(out).all()
