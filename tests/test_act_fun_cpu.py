"""Activations other than LeakyReLU (models.skip's act_fun 'Swish', 'ELU', 'none') on the host side: the module tree
against the live reference, the oracle against fixtures of the unmodified reference (tests/golden/make_act_fun.py), the
activations of the oracle and of the stage references, the stage references with each activation composed against the
oracle's autograd (tests/test_stage_ref_cpu.py's check), and the plan options of the C ABI (dip_plan_opts.act_fun).
No GPU needed."""
import ctypes
import os

import numpy as np
import pytest
import torch

import models
from oracle import dip_oracle as O
from oracle import ref_harness
import envelope_cases as E
import stage_ref as SR
from test_stage_ref_cpu import check_composed
from test_zero_pad_cpu import _desc, oracle_cfg, setup

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ["skipdefault64x96_swish", "denoise64x96_bilinear_elu", "inpaint64x96_nearest_masked_skip128_none",
         "restorekate64x96_avg_w16to128_swish"]
KINDS = ["Swish", "ELU", "none"]


def build_net(case, g):
    """the fixture's network through the public builders, called as tests/golden/make_act_fun.py calls the reference's"""
    act = str(g["act_fun"])
    if case.startswith("skipdefault"):
        return models.skip(32, 3, act_fun=act)
    if str(g["builder"]) == "get_net":
        return models.get_net(32, "skip", str(g["pad"]), str(g["modes"][0]), skip_n33d=128, skip_n33u=128,
                              skip_n11=int(g["skip_ch"]), num_scales=5, act_fun=act)
    chans, skips = [int(x) for x in g["chans"]], [int(x) for x in g["skips"]]
    return models.skip(int(g["in_depth"]), int(g["out_ch"]), num_channels_down=chans, num_channels_up=chans,
                       num_channels_skip=skips, upsample_mode=str(g["modes"][0]), downsample_mode=str(g["downsample_mode"]),
                       pad=str(g["pad"]), act_fun=act)


# ------------------------------------------------------------------------------------------------ module tree
@pytest.mark.parametrize("case", CASES)
def test_module_tree_matches_act_fixture(case):
    """state_dict keys of the reference's tree (Swish has a parameter-free `s` child), the engine spec, and the init draws
    in the oracle's parameter order"""
    g = np.load(os.path.join(GOLD, case + "_fp32.npz"))
    torch.manual_seed(0)
    net = build_net(case, g)
    assert list(net.state_dict().keys()) == [str(k) for k in g["state_keys"]]
    assert net._dip_spec is not None, net._dip_why
    assert net._dip_spec["act_fun"] == str(g["act_fun"]) and net._dip_spec["pad"] == str(g["pad"])
    for a, b in zip(net.parameters(), O.init_params(oracle_cfg(g), seed=0)):
        assert a.shape == b.shape and torch.equal(a.detach(), b.detach())


@pytest.mark.skipif(not ref_harness.available(), reason="reference checkout not present")
@pytest.mark.parametrize("act_fun", ["LeakyReLU"] + KINDS)
def test_tree_equals_live_reference(act_fun):
    """same state_dict keys, parameter order and init draws as the live reference for every act_fun string, the engine
    spec carries the string, and the stock-torch forward of the tree matches the reference's and the oracle's"""
    kw = dict(num_channels_down=[16, 32, 64, 128, 128], num_channels_up=[16, 32, 64, 128, 128], num_channels_skip=[4] * 5,
              upsample_mode="nearest", pad="reflection", act_fun=act_fun)
    with ref_harness.reference_modules() as ref:
        torch.manual_seed(11)
        rnet = ref.models.skip(32, 3, **kw)
        rsd = {k: v.clone() for k, v in rnet.state_dict().items()}
        rnames = [n for n, _ in rnet.named_parameters()]
        rmods = [type(m).__name__ for m in rnet.modules()]
        z = torch.rand(1, 32, 64, 96)
        rout = rnet(z).detach()
    torch.manual_seed(11)
    net = models.skip(32, 3, **kw)
    assert net._dip_spec is not None and net._dip_spec["act_fun"] == act_fun
    assert [n for n, _ in net.named_parameters()] == rnames
    assert [type(m).__name__ for m in net.modules()][1:] == rmods[1:]   # (the root is SkipNet here, Sequential there)
    sd = net.state_dict()
    assert list(sd.keys()) == list(rsd.keys())
    for k in sd:
        assert torch.equal(sd[k], rsd[k]), k
    models.allow_torch_execution(True)
    try:
        out = net(z).detach()
    finally:
        models.allow_torch_execution(False)
    assert torch.allclose(out, rout, atol=1e-6)
    cfg = E.cfg_of("skipdefault", act_fun=act_fun)
    assert torch.allclose(O.skip_forward(O.init_params(cfg, seed=11), z, cfg).detach(), rout, atol=1e-6)


def test_get_net_forwards_act_fun():
    for act_fun in ["LeakyReLU"] + KINDS:
        net = models.get_net(32, "skip", "reflection", "bilinear", skip_n33d=128, skip_n33u=128, skip_n11=4, num_scales=5,
                             act_fun=act_fun)
        assert net._dip_spec is not None and net._dip_spec["act_fun"] == act_fun


def test_act_fun_module_class_is_not_accelerated():
    """act_fun given as a module class (the reference calls it: models/common.py:91-92) builds the same tree but stays on
    stock torch, with a reason that names act_fun"""
    net = models.skip(32, 3, act_fun=torch.nn.ReLU)
    assert net._dip_spec is None and "act_fun" in net._dip_why
    assert any(isinstance(m, torch.nn.ReLU) for m in net.modules())
    with pytest.raises(NotImplementedError, match="act_fun"):
        net(torch.rand(1, 32, 64, 64))


# ------------------------------------------------------------------------------------------------ oracle vs reference
@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_reference_golden_fp64(case):
    g = np.load(os.path.join(GOLD, case + "_fp64.npz"))
    cfg, z0, target, mask, noises = setup(g, torch.float64)
    params = O.init_params(cfg, seed=0, dtype=torch.float64)
    rec = {}

    def record(i, out, loss, grads):
        if i == 0:
            rec["out0"], rec["grads0"] = out, [x.clone() for x in grads]

    losses, _ = O.run(cfg, params, z0, target, noises, float(g["sigma"]), float(g["lr"]), mask=mask, record=record)
    assert np.allclose(rec["out0"].numpy(), g["out0"], atol=1e-10)
    assert np.allclose(losses, g["losses"], rtol=1e-10)
    gn = np.array([x.double().norm().item() for x in rec["grads0"]])
    big = g["gnorm0"] > 1e-9
    assert np.allclose(gn[big], g["gnorm0"][big], rtol=1e-6)
    assert np.allclose(rec["grads0"][0].numpy(), g["g_skip0_w"], rtol=1e-6, atol=1e-12)
    assert np.allclose(rec["grads0"][4 if int(g["skip_ch"]) else 0].numpy(), g["g_d1_0_w"], rtol=1e-6, atol=1e-12)


@pytest.mark.parametrize("case", CASES)
def test_act_oracle_differs_from_leaky_relu(case):
    """the activations give different networks (the fixtures above would not tell a LeakyReLU oracle apart otherwise)"""
    g = np.load(os.path.join(GOLD, case + "_fp64.npz"))
    cfg, z0, _, _, noises = setup(g, torch.float64)
    params = O.init_params(cfg, seed=0, dtype=torch.float64)
    z = z0 + noises[0] * float(g["sigma"])
    assert np.abs(O.skip_forward(params, z, cfg).detach().numpy() - g["out0"]).max() < 1e-10
    cfg.act_fun = "LeakyReLU"
    assert np.abs(O.skip_forward(params, z, cfg).detach().numpy() - g["out0"]).max() > 1e-4


# ------------------------------------------------------------------------------------------------ activations
STAGE_CASES = [(k, kind, pad) for kind in KINDS for k, pad in
               (("cs4", "reflection"), ("cs4", "zero"), ("cs128", "reflection"), ("skipdefault", "zero"))] + \
              [("cs0", "Swish", "zero"), ("snail", "ELU", "reflection"), ("kate", "none", "zero"),
               ("modes_ingrad", "Swish", "reflection"), ("modes_ingrad", "ELU", "zero"), ("kate", "Swish", "reflection")]


@pytest.mark.parametrize("net,kind,pad", STAGE_CASES)
def test_composed_act_stages_reproduce_the_oracle(net, kind, pad):
    """tests/stage_ref.py with the activation and its derivative in fp64, composed stage by stage, against the oracle's
    network with the same activation and its autograd gradients (tests/test_stage_ref_cpu.py's check, which also finds
    no excluded element)"""
    check_composed(E.cfg_of(net, pad, kind), 64, 96, net == "modes_ingrad")


def test_activation_values_and_derivatives():
    """the oracle's activations against their closed forms (an unknown kind is refused), the derivative stage_ref applies
    against autograd of them, and the concat BatchNorm applies no activation"""
    y = torch.linspace(-30, 30, 601, dtype=torch.float64).reshape(-1, 1)
    expect = {"Swish": y * torch.sigmoid(y), "ELU": torch.where(y > 0, y, torch.expm1(y)), "none": y}
    for kind in KINDS:
        assert torch.allclose(O._act(y, kind), expect[kind], rtol=1e-14, atol=1e-300)
        yy = y.clone().requires_grad_(True)
        d_auto = torch.autograd.grad(O._act(yy, kind).sum(), yy)[0]
        assert torch.allclose(SR.GRAD[kind](y), d_auto, rtol=1e-12, atol=1e-300)
    for bad in ("relu", "leakyrelu", None):
        with pytest.raises(ValueError, match="act_fun"):
            O._act(y, bad)
    raw = torch.randn(6, 4, 8, dtype=torch.float64)
    g, b = torch.rand(8, dtype=torch.float64) + 0.5, torch.rand(8, dtype=torch.float64) - 0.5
    plain = SR.Bn(raw, g, b).out(act=False)
    gout = torch.randn(6, 4, 8, dtype=torch.float64)
    for kind in KINDS:   # (CatBn runs out / backward with act=False only)
        bn = SR.Bn(raw, g, b, kind)
        assert torch.equal(bn.out(act=False), plain) and torch.equal(bn.out(), SR.FWD[kind](plain))
        res = bn.backward(gout, act=False)
        assert torch.equal(res["dx"], SR.Bn(raw, g, b).backward(gout, act=False)["dx"]) and not res["excl"].any()


# ------------------------------------------------------------------------------------------------ C ABI
def test_act_fun_plan_options_workspace_query():
    """every act_fun needs the same workspace as LeakyReLU (and as NULL options), in both paddings; an unknown act_fun is
    rejected with a reason that names it"""
    import dip_engine as de
    L = de.lib()
    descs = [(_desc(de, 32, 3, 5, 128, 4, 1, 1, 0), 512, 512),                                        # denoising, tf32
             (_desc(de, 32, 3, 5, 128, 128, 0, 1, 2), 512, 512),                                      # skip=128 nearest, bf16
             (_desc(de, 32, 3, 5, 0, 0, 0, 1, 1, per_scale=([16, 32, 64, 128, 128], [4] * 5)), 64, 96),  # skip() default, fp32
             (_desc(de, 32, 3, 5, 0, 0, 1, 1, 0, per_scale=([16, 32, 64, 128, 128], [0] * 5), dmode=1), 64, 96),
             (_desc(de, 3, 1, 5, 128, 4, 1, 0, 0, 0, 1), 64, 96)]                                     # input_grad, logits
    kinds = [de.ACT_LEAKY_RELU, de.ACT_SWISH, de.ACT_ELU, de.ACT_NONE]
    assert kinds == [0, 1, 2, 3] and [de.ACT_FUNS[k] for k in ("LeakyReLU", "Swish", "ELU", "none")] == kinds
    for d, H_, W_ in descs:
        null = L.dip_plan_workspace_bytes_opts(ctypes.byref(d), H_, W_, None)
        sizes = [L.dip_plan_workspace_bytes_opts(ctypes.byref(d), H_, W_, ctypes.byref(de.PlanOpts(pad, act)))
                 for pad in (de.PAD_REFLECTION, de.PAD_ZERO) for act in kinds]
        assert null > 0 and all(n == null for n in sizes), (null, sizes)
    d = descs[0][0]
    for bad in (4, -1, 100):
        for pad in (de.PAD_REFLECTION, de.PAD_ZERO):
            n = L.dip_plan_workspace_bytes_opts(ctypes.byref(d), 512, 512, ctypes.byref(de.PlanOpts(pad, bad)))
            assert n == 0 and b"act_fun" in L.dip_last_error(), L.dip_last_error()
    # a bad pad_mode is still reported as such
    assert L.dip_plan_workspace_bytes_opts(ctypes.byref(d), 512, 512, ctypes.byref(de.PlanOpts(2, de.ACT_SWISH))) == 0
    assert b"pad_mode" in L.dip_last_error()


def test_plan_opts_layout():
    """dip_plan_opts is {pad_mode, act_fun}; the positional PlanOpts(pad) of the zero-pad callers means LeakyReLU"""
    import dip_engine as de
    assert [f for f, _ in de.PlanOpts._fields_] == ["pad_mode", "act_fun"] and ctypes.sizeof(de.PlanOpts) == 8
    o = de.PlanOpts(de.PAD_ZERO)
    assert (o.pad_mode, o.act_fun) == (de.PAD_ZERO, de.ACT_LEAKY_RELU)
    o = de.PlanOpts()
    assert (o.pad_mode, o.act_fun) == (de.PAD_REFLECTION, de.ACT_LEAKY_RELU)


@pytest.mark.parametrize("bad", ["relu", "leakyrelu", "Sigmoid", None, torch.nn.ReLU])
def test_plan_rejects_unknown_act_before_touching_the_device(bad):
    import dip_engine as de
    with pytest.raises(ValueError, match="act"):
        de.Plan(32, 3, 5, 128, 4, True, 64, 96, act=bad)


def test_engine_spec_routes_act_fun():
    """_dip_spec carries the act_fun string (SkipNet builds its plan with it)"""
    for act_fun in ["LeakyReLU"] + KINDS:
        net = models.skip(32, 3, act_fun=act_fun)
        assert net._dip_spec["act_fun"] == act_fun and net._dip_why is None
