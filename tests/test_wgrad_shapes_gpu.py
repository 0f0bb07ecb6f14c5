"""Tensor-core weight gradient (dip_op_conv_wgrad) at the shapes the 512x512 flagship step runs, vs an fp64 reference
computed on the GPU (one GEMM per filter tap).

tf32 mode: <= 2e-3 relative Frobenius error.  bf16 mode: the reference is evaluated on the operands rounded to bf16, so
only the fp32 accumulation differs: <= 2e-5.  bf16 runs at the shapes whose bf16 operand copies fit in the single-op
scratch area (96 MB).  Every case is run twice: the gradient must be bitwise the same (split-K partials summed in a fixed
order).
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = {0: 2e-3, 2: 2e-5}

# (C, k, stride, out_h, out_w, rot)
L0_UP = (132, 3, 1, 512, 512, 4)       # level-0 3x3 up conv on the 128 + 4 channel concat: 136 accumulator columns
L0_1X1 = (128, 1, 1, 512, 512, 0)
L0_DOWN1 = (32, 3, 2, 256, 256, 0)     # level-0 3x3 stride-2 down conv on the 32-channel input
L1_DOWN2 = (128, 3, 1, 256, 256, 0)
L1_UP = (132, 3, 1, 256, 256, 4)
RAGGED = (132, 3, 1, 100, 300, 4)      # width not a multiple of the 32-pixel block

CASES = [(L0_UP, 0), (L0_1X1, 0), (L0_DOWN1, 0), (L1_DOWN2, 0), (RAGGED, 0),
         (L0_DOWN1, 2), (L1_DOWN2, 2), (L1_UP, 2), (RAGGED, 2)]


def ref_wgrad(dy, a, k, stride):
    """dW[n][c][r][s] = sum_pixels dY[n][y][x] * A[c][stride*y + r][stride*x + s], fp64, one GEMM per tap"""
    n, oh, ow = dy.shape
    C = a.shape[0]
    y = dy.reshape(n, -1)
    dw = torch.empty(n, C, k, k, dtype=torch.float64, device=dy.device)
    for r in range(k):
        for s in range(k):
            x = a[:, r:r + stride * (oh - 1) + 1:stride, s:s + stride * (ow - 1) + 1:stride].reshape(C, -1)
            dw[:, :, r, s] = y @ x.T
    return dw


@pytest.mark.parametrize("case,prec", CASES, ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else
                         {0: "tf32", 2: "bf16"}[v])
def test_wgrad_flagship_shapes(case, prec):
    import dip_engine as de
    C, k, stride, oh, ow, rot = case
    g = torch.Generator(device="cuda").manual_seed(5)
    ih, iw = (oh - 1) * stride + k, (ow - 1) * stride + k
    if stride == 2:  # engine buffers are padded to even extents
        ih += ih % 2
        iw += iw % 2
    a = torch.randn(ih, iw, C, generator=g, device="cuda")       # NHWC
    dy = torch.randn(oh, ow, 128, generator=g, device="cuda")
    dw = de.op_conv_wgrad(dy, a, C, k, stride, 0, 0, rot=rot, precision=prec)
    dw2 = de.op_conv_wgrad(dy, a, C, k, stride, 0, 0, rot=rot, precision=prec)
    torch.cuda.synchronize()
    assert torch.equal(dw, dw2)

    def opnd(x):   # the operand as the kernel reads it, in fp64, channels first
        return (x.bfloat16() if prec == 2 else x).double().permute(2, 0, 1)

    ref = ref_wgrad(opnd(dy), torch.roll(opnd(a), rot, 0), k, stride)
    err = ((dw.double() - ref).norm() / ref.norm()).item()
    assert err < TOL[prec], err
