"""Small-shape launches of every hand-written mbarrier / TMA / wgmma kernel for compute-sanitizer (SURVEY.md 5, 7.3.3):
  compute-sanitizer --tool memcheck|racecheck|synccheck python scripts/sanitize_ops.py
Covers tc_conv_kernel (1x1, 3x3, stride 2, N split, K tail with C=132, several waves of ragged tiles, 4-phase stride-2
dgrad), tc_conv_patch_kernel (stride-1 3x3: ragged tiles, one tile, N split 2 and 4, K tail), tc_wgrad_kernel (split-K partials, in-smem operand transpose) and one full forward + backward + Adam step of the
engine at 64x64.  Without the sanitizer it runs as a plain parity check (relative errors vs torch-CPU fp64).
DIP_SAN_PREC=2 runs the same launches in the bf16 mode (tc_conv_kernel_bf16 / tc_wgrad_kernel_bf16, bf16 twins written by the
producer kernels); DIP_SAN_NARROW=1 adds a step of the per-scale-width network (snail) with 'avg' downsampling."""
import os
import sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "deep-image-prior_b200"))
import torch
import torch.nn.functional as F
import dip_engine as de


def nhwc(x):
    return x.permute(1, 2, 0).contiguous()


def rel(a, b):
    return ((a.double().cpu() - b.double()).norm() / b.double().norm()).item()


PREC = int(os.environ.get("DIP_SAN_PREC", "0"))
g = torch.Generator().manual_seed(0)
# (C, k, stride, oh, ow): 1x1, 3x3 (N split), stride 2, K tail (C=132), several waves of ragged tiles; stride-1 3x3 patch
# path: ragged 8x16 tiles, a single tile (N split 4), N split 2, K tail with ragged tiles
for C, k, stride, oh, ow in [(128, 1, 1, 32, 32), (128, 3, 1, 16, 16), (32, 3, 2, 32, 32), (132, 3, 1, 40, 24), (128, 3, 1, 270, 150),
                             (128, 3, 1, 37, 21), (128, 3, 1, 16, 8), (128, 3, 1, 80, 80), (132, 3, 1, 45, 30)]:
    ih, iw = (oh - 1) * stride + k, (ow - 1) * stride + k
    ih += ih % 2 if stride == 2 else 0
    iw += iw % 2 if stride == 2 else 0
    a = torch.randn(C, ih, iw, generator=g)
    w = torch.randn(128, C, k, k, generator=g) / (C * k * k) ** 0.5
    b = torch.randn(128, generator=g)
    stats = torch.zeros(256 * 16, dtype=torch.float64, device="cuda")
    d = de.op_conv_fprop(nhwc(a).cuda(), w.cuda(), b.cuda(), k, stride, 0, 0, oh, ow, stats=stats, precision=PREC)
    ref = F.conv2d(a[None].double(), w.double(), b.double(), stride=stride)[0][:, :oh, :ow]
    print("fprop C=%d k=%d s=%d %dx%d rel err %.2e" % (C, k, stride, oh, ow, rel(d.permute(2, 0, 1), ref)))
    dy = torch.randn(128, oh, ow, generator=g)
    dw = de.op_conv_wgrad(nhwc(dy).cuda(), nhwc(a).cuda(), C, k, stride, 0, 0, precision=PREC)
    refw = torch.nn.grad.conv2d_weight(a[None, :, :(oh - 1) * stride + k, :(ow - 1) * stride + k].double(), (128, C, k, k),
                                       dy[None].double(), stride=stride)
    print("wgrad rel err %.2e" % rel(dw, refw))
    if stride == 1:
        dx = de.op_conv_dgrad(nhwc(dy).cuda(), w.cuda(), k, oh + k - 1, ow + k - 1, precision=PREC)
        print("dgrad rel err %.2e" % rel(dx.permute(2, 0, 1), F.conv_transpose2d(dy[None].double(), w.double())[0]))
dy = torch.randn(128, 20, 12, generator=g)
w = torch.randn(128, 128, 3, 3, generator=g) / 34.
dx = de.op_conv_dgrad_s2(nhwc(dy).cuda(), w.cuda(), precision=PREC)
print("dgrad s2 rel err %.2e" % rel(dx.permute(2, 0, 1)[:, :41, :25], F.conv_transpose2d(dy[None].double(), w.double(), stride=2)[0]))
# one full step of the engine (graph replay off: the sanitizer then sees every launch in stream order)
os.environ["DIP_NO_GRAPH"] = "1"
from oracle import dip_oracle as O
plan = de.Plan(32, 3, 5, 128, 4, True, 64, 64, precision=PREC)
params = [p.detach().cuda().contiguous() for p in O.init_params(O.SkipConfig(), seed=0)]
grads = [torch.zeros_like(p) for p in params]
plan.bind(params, grads)
for p, gb in zip(params, grads):
    p.grad = gb
adam = de.FusedAdam(params, lr=0.01)
adam._bind(grads)
hist = torch.zeros(2, dtype=torch.float64, device="cuda")
de.run_iterations(plan, adam, torch.rand(1, 32, 64, 64, device="cuda") * 0.1, torch.rand(1, 3, 64, 64, device="cuda"), None,
                  1. / 30, 1, 2, 0.01, loss_hist=hist)
torch.cuda.synchronize()
print("engine step losses", hist.tolist())
if os.environ.get("DIP_SAN_NARROW") is not None:
    cfg = O.SkipConfig(in_channels=3, channels=[8, 16, 32, 64, 128], skip_channels=[0, 0, 0, 4, 4])
    cfg.downsample_mode = "avg"
    plan = de.Plan(3, 3, 5, cfg.channels, cfg.skip_channels, True, 64, 96, precision=PREC, downsample_mode="avg")
    params = [p.detach().cuda().contiguous() for p in O.init_params(cfg, seed=0)]
    grads = [torch.zeros_like(p) for p in params]
    plan.bind(params, grads)
    for p, gb in zip(params, grads):
        p.grad = gb
    adam = de.FusedAdam(params, lr=0.01)
    adam._bind(grads)
    de.run_iterations(plan, adam, torch.rand(1, 3, 64, 96, device="cuda") * 0.1, torch.rand(1, 3, 64, 96, device="cuda"), None,
                      1. / 30, 1, 2, 0.01, loss_hist=hist)
    torch.cuda.synchronize()
    print("narrow (snail widths, avg downsampling) engine step losses", hist.tolist())
