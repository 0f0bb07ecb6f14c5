"""The fp64 stage references of tests/stage_ref.py, composed stage by stage, against the oracle's whole network and its
autograd gradients (CPU only).  This checks the layout, the concat rotation, the pads and folds, the activations and
their derivatives, the skip-conv terms and the upsampling adjoints of the references before they judge the engine
(tests/test_stages_gpu.py, tests/test_envelope_gpu.py).  `check_composed` is the one composition check; the zero-padded
networks (tests/test_zero_pad_cpu.py), the other activations (tests/test_act_fun_cpu.py) and the envelope rows
(tests/test_envelope_cpu.py) run it too."""
import pytest
import torch

from oracle import dip_oracle as O
import envelope_cases as E
import stage_ref as SR

H, W = 64, 96


def compose(cfg, params, z, target, input_grad):
    refs = SR.Refs()

    def src(name):
        if name.startswith("L") and name.endswith(".Pin") and name != "L0.Pin":   # a level's input = the level above's P_d2
            name = "L%d.P_d2" % (int(name[1:-4]) - 1)
        return refs[name]

    SR.forward(cfg, params, src, "fp64", refs, z=z)
    out = refs["out"]
    dout = 2.0 * (out - target[0]) / out.numel()
    SR.backward(cfg, params, src, "fp64", refs, dout, input_grad=input_grad)
    return refs


def check_composed(cfg, H, W, input_grad):
    """cfg's stage references composed stage by stage (fp64, random affine parameters) against the oracle's output and
    autograd gradients, dz with input_grad; with every structural check that applies to cfg"""
    params = SR.random_affine(cfg, O.init_params(cfg, seed=0, dtype=torch.float64), seed=7)
    g = torch.Generator().manual_seed(3)
    z = torch.rand(1, cfg.in_channels, H, W, generator=g, dtype=torch.float64)
    target = torch.rand(1, cfg.out_channels, H, W, generator=g, dtype=torch.float64)
    refs = compose(cfg, params, z, target, input_grad)
    pin = refs["L0.Pin"]   # the stored depth's channels after the real ones are zeros
    assert pin.shape[-1] == SR.stored_depth(cfg, 0) and pin[..., cfg.in_channels:].abs().sum().item() == 0
    if cfg.pad != "reflection":   # a zero halo ring
        assert pin[0].abs().max() == 0 and pin[-1].abs().max() == 0 and pin[:, 0].abs().max() == 0 and pin[:, -1].abs().max() == 0
    if cfg.act_fun != "LeakyReLU":   # no jump in the derivative: no element is excluded from the backward checks
        assert refs.excl and all(frac == 0 for frac, _ in refs.excl.values())
        assert all(e is None or not e.any() for _, _, e in refs.d.values())

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


@pytest.mark.parametrize("kind", ["cs4", "cs128", "cs0", "snail", "kate", "modes_ingrad"])
def test_composed_stages_reproduce_the_oracle(kind):
    check_composed(E.cfg_of(kind), H, W, kind == "modes_ingrad")
