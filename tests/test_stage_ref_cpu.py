"""The fp64 stage references of tests/stage_ref.py, composed stage by stage, against the oracle's whole network and its
autograd gradients (CPU only).  This checks the layout, the concat rotation, the folds, the skip-conv terms and the
upsampling adjoints of the references before they judge the engine (tests/test_stages_gpu.py)."""
import re

import pytest
import torch

from oracle import dip_oracle as O
import stage_ref as SR

H, W = 64, 96


def cfg_of(kind):
    if kind == "cs4":
        return O.SkipConfig(skip_channels=4, upsample_mode="bilinear")
    if kind == "cs128":
        return O.SkipConfig(skip_channels=128, upsample_mode="nearest")
    if kind == "cs0":
        return O.SkipConfig(skip_channels=0, upsample_mode="bilinear")
    if kind == "snail":
        return O.SkipConfig(in_channels=3, channels=[8, 16, 32, 64, 128], skip_channels=[0, 0, 0, 4, 4])
    if kind == "kate":
        c = O.SkipConfig(in_channels=3, channels=[16, 32, 64, 128, 128], skip_channels=0)
        c.downsample_mode = "avg"
        return c
    if kind == "modes_ingrad":   # per-scale upsampling, logits as the output, one output channel, dL/d(input)
        return O.SkipConfig(in_channels=3, out_channels=1, skip_channels=4, need_sigmoid=False,
                            upsample_mode=["bilinear", "nearest", "bilinear", "nearest", "nearest"])
    raise KeyError(kind)


def compose(cfg, params, z, target, input_grad):
    refs = SR.Refs()

    def src(name):
        m = re.match(r"L(\d+)\.Pin$", name)
        if m and int(m.group(1)) > 0:   # a level's input is the padded output of the level above
            name = "L%d.P_d2" % (int(m.group(1)) - 1)
        return refs[name]

    SR.forward(cfg, params, src, "fp64", refs, z=z)
    out = refs["out"]
    dout = 2.0 * (out - target[0]) / out.numel()
    SR.backward(cfg, params, src, "fp64", refs, dout, input_grad=input_grad)
    return refs


@pytest.mark.parametrize("kind", ["cs4", "cs128", "cs0", "snail", "kate", "modes_ingrad"])
def test_composed_stages_reproduce_the_oracle(kind):
    cfg = cfg_of(kind)
    input_grad = kind == "modes_ingrad"
    params = SR.random_affine(cfg, O.init_params(cfg, seed=0, dtype=torch.float64), seed=7)
    g = torch.Generator().manual_seed(3)
    z = torch.rand(1, cfg.in_channels, H, W, generator=g, dtype=torch.float64)
    target = torch.rand(1, cfg.out_channels, H, W, generator=g, dtype=torch.float64)
    refs = compose(cfg, params, z, target, input_grad)

    p = [x.detach().clone().requires_grad_(True) for x in params]
    zz = z.clone().requires_grad_(input_grad)
    out = O.skip_forward(p, zz, cfg)
    assert (refs["out"] - out.detach()[0]).abs().max().item() < 1e-12
    grads = torch.autograd.grad(O.mse_loss(out, target), p + ([zz] if input_grad else []))
    names = [n for n, _ in O.param_layout(cfg)] + (["dz"] if input_grad else [])
    gmax = max(gr.abs().max().item() for gr in grads)
    for name, gr in zip(names, grads):
        got = refs[name if name == "dz" else "grad:" + name].reshape(gr.shape)
        # (conv biases in front of a BatchNorm and the concat BN's beta have a zero gradient in exact arithmetic: the
        # floor keeps their fp64 rounding noise from counting as a relative error)
        err = (got - gr).abs().max().item()
        assert err <= max(1e-10 * gr.abs().max().item(), 1e-13 * gmax), (name, err, gr.abs().max().item())
        if SR.is_dead_bias(name):
            assert got.abs().max().item() == 0, name
        if name.endswith(".w") and name != "head.w":   # every conv weight gradient carries a Frobenius bound
            assert "grad:" + name in refs.conv, name
