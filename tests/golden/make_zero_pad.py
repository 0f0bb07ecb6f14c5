"""Generates the zero-padding fixtures tests/golden/*_zeropad_fp64.npz / *_zeropad_fp32.npz by running the UNMODIFIED
reference (imported from /root/reference) on torch-CPU.

Run in the build container only:  python tests/golden/make_zero_pad.py
Same protocol and fields as make_golden.run_variant (seeded image input, 3 Adam steps, first-step output / loss /
gradient norms / the level-0 conv gradients), plus `pad`; the input itself is not stored (the tests redraw it from the same
seeded generator).  The networks are built with pad='zero', the default of the
reference's models.skip (models/skip.py:10): every 3x3 conv is Conv2d(padding=1) without a ReflectionPad2d in front
(models/common.py:114-120).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_harness  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))

# name -> (H, W, in_depth, skip() keyword arguments beyond (in_depth, 3), sigma, masked)
CASES = {
    # models.skip(32, 3) with every other argument at its default: widths [16, 32, 64, 128, 128], skips 4, 3/3/1 filters,
    # nearest, stride, LeakyReLU, pad='zero'
    "skipdefault64x96_zeropad": (64, 96, 32, dict(), 0.03, False),
    # inpainting.ipynb kate's 128-wide skip=128 nearest network, masked loss
    "inpaint64x96_nearest_masked_skip128_zeropad": (64, 96, 32, dict(
        num_channels_down=[128] * 5, num_channels_up=[128] * 5, num_channels_skip=[128] * 5, upsample_mode="nearest",
        pad="zero"), 0.03, True),
    # restoration.ipynb kate: per-scale widths, no skips, 'avg' downsampling, masked loss
    "restorekate64x96_avg_w16to128_zeropad": (64, 96, 32, dict(
        num_channels_down=[16, 32, 64, 128, 128], num_channels_up=[16, 32, 64, 128, 128], num_channels_skip=[0] * 5,
        upsample_mode="bilinear", downsample_mode="avg", pad="zero"), 0.0, True),
}
DEFAULTS = dict(num_channels_down=[16, 32, 64, 128, 128], num_channels_skip=[4] * 5, upsample_mode="nearest",
                downsample_mode="stride", pad="zero")


def run(name, H, W, in_depth, kw, sigma, masked, dtype, iters=3, lr=0.01, out_ch=3, threads=8):
    torch.set_num_threads(threads)
    with ref_harness.reference_modules() as ref:
        torch.manual_seed(0)
        net = ref.models.skip(in_depth, out_ch, **kw).type(dtype)
        g = torch.Generator().manual_seed(2)
        z0 = torch.rand(1, in_depth, H, W, generator=g).type(dtype)
        target = torch.rand(1, out_ch, H, W, generator=g).type(dtype)
        mask = (torch.rand(1, 1, H, W, generator=g) > 0.5).type(dtype) if masked else None
        gn = torch.Generator().manual_seed(123)
        mse = torch.nn.MSELoss()
        params = [p for p in net.parameters()]
        opt = torch.optim.Adam(params, lr=lr)
        losses = []
        a = dict(DEFAULTS, **kw)
        skips = list(a["num_channels_skip"])
        for i in range(iters):
            noise = torch.randn(z0.shape, generator=gn).type(dtype)
            opt.zero_grad()
            out = net(z0 + noise * sigma)
            loss = mse(out * mask, target * mask) if masked else mse(out, target)
            loss.backward()
            if i == 0:
                out0 = out.detach().clone()
                gnorm0 = np.array([p.grad.double().norm().item() for p in params])
                g_first = [params[k].grad.detach().clone().numpy() for k in (0, 4 if skips[0] else 0)]   # L0 skip conv w, L0 down conv w
            losses.append(loss.item())
            opt.step()
        keys = list(net.state_dict().keys())
    mode = a["upsample_mode"]
    np.savez_compressed(os.path.join(HERE, name + ".npz"), H=H, W=W, in_depth=in_depth, out_ch=out_ch,
                        modes=np.array([mode] * 5), iters=iters, sigma=sigma, lr=lr, masked=masked, losses=np.array(losses),
                        out0=out0.numpy(), gnorm0=gnorm0, g_skip0_w=g_first[0], g_d1_0_w=g_first[1], dtype=str(dtype),
                        state_keys=np.array(keys), skip_ch=skips[0], chans=np.array(a["num_channels_down"]),
                        skips=np.array(skips), downsample_mode=a["downsample_mode"], pad=a["pad"])
    print(name, "losses", losses)


if __name__ == "__main__":
    for name in (sys.argv[1:] or list(CASES)):
        for dt, tag in ((torch.float64, "fp64"), (torch.float32, "fp32")):
            run(name + "_" + tag, *CASES[name], dtype=dt)
