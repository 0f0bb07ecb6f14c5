"""Generates the activation fixtures tests/golden/*_{swish,elu,none}_fp64.npz / *_fp32.npz by running the UNMODIFIED reference
(imported from /root/reference) on torch-CPU.

Run in the build container only:  python tests/golden/make_act_fun.py
Same protocol and fields as make_zero_pad.py (seeded image input, 3 Adam steps, first-step output / loss / gradient norms /
the level-0 conv gradients; the input itself is not stored, the tests redraw it from the same seeded generator), plus
`act_fun` and `builder` ('skip' or 'get_net').  Each activation of the reference's act() (models/common.py:76-92) other
than LeakyReLU meets a different network, and both paddings occur.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_harness  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))

# name -> (H, W, in_depth, builder, keyword arguments, sigma, masked)
CASES = {
    # models.skip(32, 3, act_fun='Swish'), every other argument at its default: widths [16, 32, 64, 128, 128], skips 4,
    # nearest, stride, pad='zero'
    "skipdefault64x96_swish": (64, 96, 32, "skip", dict(act_fun="Swish"), 0.03, False),
    # denoising.ipynb's get_net call (the 128-wide cs=4 bilinear reflection network) with act_fun='ELU'
    "denoise64x96_bilinear_elu": (64, 96, 32, "get_net", dict(
        NET_TYPE="skip", pad="reflection", upsample_mode="bilinear", skip_n33d=128, skip_n33u=128, skip_n11=4, num_scales=5,
        act_fun="ELU"), 0.03, False),
    # inpainting.ipynb kate's 128-wide skip=128 nearest network, masked loss, no activation
    "inpaint64x96_nearest_masked_skip128_none": (64, 96, 32, "skip", dict(
        num_channels_down=[128] * 5, num_channels_up=[128] * 5, num_channels_skip=[128] * 5, upsample_mode="nearest",
        pad="reflection", act_fun="none"), 0.03, True),
    # restoration.ipynb kate: per-scale widths, no skips, 'avg' downsampling, masked loss
    "restorekate64x96_avg_w16to128_swish": (64, 96, 32, "skip", dict(
        num_channels_down=[16, 32, 64, 128, 128], num_channels_up=[16, 32, 64, 128, 128], num_channels_skip=[0] * 5,
        upsample_mode="bilinear", downsample_mode="avg", pad="reflection", act_fun="Swish"), 0.0, True),
}
DEFAULTS = dict(num_channels_down=[16, 32, 64, 128, 128], num_channels_skip=[4] * 5, upsample_mode="nearest",
                downsample_mode="stride", pad="zero")


def skip_args(builder, kw):
    """the arguments models.skip receives (get_net forwards its own: reference models/__init__.py:8-17)"""
    if builder == "get_net":
        n = kw["num_scales"]
        return dict(num_channels_down=[kw["skip_n33d"]] * n, num_channels_skip=[kw["skip_n11"]] * n,
                    upsample_mode=kw["upsample_mode"], downsample_mode="stride", pad=kw["pad"], act_fun=kw["act_fun"])
    return dict(DEFAULTS, **kw)


def run(name, H, W, in_depth, builder, kw, sigma, masked, dtype, iters=3, lr=0.01, out_ch=3, threads=8):
    torch.set_num_threads(threads)
    with ref_harness.reference_modules() as ref:
        torch.manual_seed(0)
        if builder == "get_net":
            net = ref.models.get_net(in_depth, n_channels=out_ch, **kw).type(dtype)
        else:
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
        a = skip_args(builder, kw)
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
                        skips=np.array(skips), downsample_mode=a["downsample_mode"], pad=a["pad"], act_fun=a["act_fun"],
                        builder=builder)
    print(name, "losses", losses)


if __name__ == "__main__":
    for name in (sys.argv[1:] or list(CASES)):
        for dt, tag in ((torch.float64, "fp64"), (torch.float32, "fp32")):
            run(name + "_" + tag, *CASES[name], dtype=dt)
