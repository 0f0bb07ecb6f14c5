"""Zero padding (models.skip's default pad='zero', and every other value that is not 'reflection') on the host side:
the module tree against the reference, the oracle against fixtures of the unmodified reference
(tests/golden/make_zero_pad.py), the zero pad of the stage references and its adjoint, the zero-padded stage references
composed against the oracle's autograd (tests/test_stage_ref_cpu.py's check), and the plan options of the C ABI
(dip_plan_opts).  No GPU needed."""
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

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ["skipdefault64x96_zeropad", "inpaint64x96_nearest_masked_skip128_zeropad", "restorekate64x96_avg_w16to128_zeropad"]


def oracle_cfg(g):
    """the oracle's SkipConfig of a zero-pad or act_fun fixture"""
    chans, skips = [int(x) for x in g["chans"]], [int(x) for x in g["skips"]]
    modes = [str(m) for m in g["modes"]]
    if set(chans) == {128} and len(set(skips)) == 1:
        cfg = O.SkipConfig(in_channels=int(g["in_depth"]), out_channels=int(g["out_ch"]), upsample_mode=modes, skip_channels=skips[0])
    else:
        cfg = O.SkipConfig(in_channels=int(g["in_depth"]), out_channels=int(g["out_ch"]), upsample_mode=modes, channels=chans,
                           skip_channels=skips)
    cfg.downsample_mode = str(g["downsample_mode"])
    cfg.pad = str(g["pad"])
    if "act_fun" in g.files:
        cfg.act_fun = str(g["act_fun"])
    return cfg


def setup(g, dtype):
    """the fixture's inputs, drawn as tests/golden/make_zero_pad.py and make_act_fun.py draw them"""
    cfg = oracle_cfg(g)
    H_, W_ = int(g["H"]), int(g["W"])
    gen = torch.Generator().manual_seed(2)
    z0 = torch.rand(1, cfg.in_channels, H_, W_, generator=gen).to(dtype)
    target = torch.rand(1, cfg.out_channels, H_, W_, generator=gen).to(dtype)
    mask = (torch.rand(1, 1, H_, W_, generator=gen) > 0.5).to(dtype) if bool(g["masked"]) else None
    gn = torch.Generator().manual_seed(123)
    noises = [torch.randn(z0.shape, generator=gn).to(dtype) for _ in range(int(g["iters"]))]
    return cfg, z0, target, mask, noises


def build_skip(g):
    """models.skip with the fixture's arguments"""
    chans, skips = [int(x) for x in g["chans"]], [int(x) for x in g["skips"]]
    return models.skip(int(g["in_depth"]), int(g["out_ch"]), num_channels_down=chans, num_channels_up=chans,
                       num_channels_skip=skips, upsample_mode=str(g["modes"][0]), downsample_mode=str(g["downsample_mode"]),
                       pad=str(g["pad"]))


# ------------------------------------------------------------------------------------------------ module tree
def test_default_skip_is_accelerated_with_zero_padding():
    net = models.skip()
    assert net._dip_spec is not None and net._dip_spec["pad"] == "zero", net._dip_why
    assert not any(isinstance(m, torch.nn.ReflectionPad2d) for m in net.modules())
    net = models.get_net(32, "skip", "zero", "nearest", skip_n33d=128, skip_n33u=128, skip_n11=4, num_scales=5)
    assert net._dip_spec is not None and net._dip_spec["pad"] == "zero"
    net = models.get_net(32, "skip", "reflection", "bilinear", skip_n33d=128, skip_n33u=128, skip_n11=4, num_scales=5)
    assert net._dip_spec["pad"] == "reflection"


@pytest.mark.parametrize("case", CASES)
def test_module_tree_matches_zero_pad_fixture(case):
    """state_dict keys of the reference's tree (no ReflectionPad2d children: keys shift), and the init draws in the
    oracle's parameter order"""
    g = np.load(os.path.join(GOLD, case + "_fp32.npz"))
    torch.manual_seed(0)
    net = models.skip(32, 3) if case.startswith("skipdefault") else build_skip(g)
    assert list(net.state_dict().keys()) == [str(k) for k in g["state_keys"]]
    assert net._dip_spec is not None and net._dip_spec["pad"] == "zero"
    assert net._dip_spec["downsample_mode"] == str(g["downsample_mode"])
    for a, b in zip(net.parameters(), O.init_params(oracle_cfg(g), seed=0)):
        assert a.shape == b.shape and torch.equal(a.detach(), b.detach())


@pytest.mark.skipif(not ref_harness.available(), reason="reference checkout not present")
@pytest.mark.parametrize("pad", ["zero", "replication"])
def test_tree_equals_live_reference(pad):
    """any pad other than 'reflection' is zero padding in the reference (models/common.py:114-120): same state_dict keys,
    parameter order and init draws as the live reference, the engine spec says 'zero', and the stock-torch forward of
    the tree matches the reference's"""
    kw = dict(num_channels_down=[16, 32, 64, 128, 128], num_channels_up=[16, 32, 64, 128, 128], num_channels_skip=[4] * 5,
              upsample_mode="nearest", pad=pad)
    with ref_harness.reference_modules() as ref:
        torch.manual_seed(11)
        rnet = ref.models.skip(32, 3, **kw)
        rsd = {k: v.clone() for k, v in rnet.state_dict().items()}
        rnames = [n for n, _ in rnet.named_parameters()]
        z = torch.rand(1, 32, 64, 96)
        rout = rnet(z).detach()
    torch.manual_seed(11)
    net = models.skip(32, 3, **kw)
    assert net._dip_spec is not None and net._dip_spec["pad"] == "zero"
    assert [n for n, _ in net.named_parameters()] == rnames
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
    cfg = E.cfg_of("skipdefault", "zero")
    assert torch.allclose(O.skip_forward(O.init_params(cfg, seed=11), z, cfg).detach(), rout, atol=1e-6)


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


def test_zero_pad_oracle_differs_from_reflection():
    """the two paddings give different networks (the fixtures above would not tell a reflection oracle apart otherwise)"""
    g = np.load(os.path.join(GOLD, CASES[0] + "_fp64.npz"))
    cfg, z0, _, _, noises = setup(g, torch.float64)
    params = O.init_params(cfg, seed=0, dtype=torch.float64)
    z = z0 + noises[0] * float(g["sigma"])
    assert np.abs(O.skip_forward(params, z, cfg).detach().numpy() - g["out0"]).max() < 1e-10
    cfg.pad = "reflection"
    assert np.abs(O.skip_forward(params, z, cfg).detach().numpy() - g["out0"]).max() > 1e-4


# ------------------------------------------------------------------------------------------------ stage references
@pytest.mark.parametrize("kind", ["cs4", "cs128", "cs0", "snail", "kate", "modes_ingrad", "skipdefault"])
def test_composed_zero_pad_stages_reproduce_the_oracle(kind):
    """tests/stage_ref.py with zero padding (zero halos, folds that drop the halo), composed stage by stage, against the
    oracle's zero-padded network and its autograd gradients (tests/test_stage_ref_cpu.py's check)"""
    check_composed(E.cfg_of(kind, "zero"), 64, 96, kind == "modes_ingrad")


def test_zero_pad_and_its_fold():
    """stage_ref pads every value of pad other than 'reflection' with a zero halo, and its fold keeps the interior"""
    x = torch.rand(4, 6, 3, dtype=torch.float64)
    assert SR.padding(O.SkipConfig()) == (SR.reflect_pad, SR.fold)
    for pad in ("zero", "replication"):
        p, fold = SR.padding(E.cfg_of("cs4", pad))
        y = p(x)
        ring = torch.ones(6, 8, 1, dtype=torch.bool)
        ring[1:-1, 1:-1] = False
        assert torch.equal(y[1:-1, 1:-1], x) and (y * ring).abs().max() == 0 and torch.equal(fold(y), x)


# ------------------------------------------------------------------------------------------------ C ABI
def _desc(de, *args, per_scale=None, dmode=0):
    d = de.NetDesc(*args)
    if per_scale is not None:
        for i, (a, c) in enumerate(zip(*per_scale)):
            d.channels_down[i], d.channels_up[i], d.channels_skip[i] = a, a, c
    d.downsample_mode = dmode
    return d


def test_plan_options_workspace_query():
    """zero padding is accepted and needs the same workspace as reflection; an unknown pad_mode is rejected with a
    reason; NULL options are the plain query"""
    import dip_engine as de
    L = de.lib()
    for sym in ("dip_plan_workspace_bytes_opts", "dip_plan_create_opts"):
        assert hasattr(L, sym) and sym in de.ABI_SYMBOLS
    descs = [(_desc(de, 32, 3, 5, 128, 4, 1, 1, 0), 512, 512),                                        # denoising, tf32
             (_desc(de, 32, 3, 5, 128, 128, 0, 1, 2), 512, 512),                                      # skip=128 nearest, bf16
             (_desc(de, 32, 3, 5, 0, 0, 0, 1, 1, per_scale=([16, 32, 64, 128, 128], [4] * 5)), 64, 96),  # skip() default, fp32
             (_desc(de, 32, 3, 5, 0, 0, 1, 1, 0, per_scale=([16, 32, 64, 128, 128], [0] * 5), dmode=1), 64, 96),
             (_desc(de, 3, 1, 5, 128, 4, 1, 0, 0, 0, 1), 64, 96)]                                     # input_grad, logits
    for d, H_, W_ in descs:
        plain = L.dip_plan_workspace_bytes(ctypes.byref(d), H_, W_)
        refl = L.dip_plan_workspace_bytes_opts(ctypes.byref(d), H_, W_, ctypes.byref(de.PlanOpts(de.PAD_REFLECTION)))
        zero = L.dip_plan_workspace_bytes_opts(ctypes.byref(d), H_, W_, ctypes.byref(de.PlanOpts(de.PAD_ZERO)))
        null = L.dip_plan_workspace_bytes_opts(ctypes.byref(d), H_, W_, None)
        assert plain > 0 and plain == refl == zero == null, (plain, refl, zero, null)
    d = descs[0][0]
    for bad in (2, -1):
        n = L.dip_plan_workspace_bytes_opts(ctypes.byref(d), 512, 512, ctypes.byref(de.PlanOpts(bad)))
        assert n == 0 and b"pad" in L.dip_last_error()
    # an unsupported network in zero mode is still refused for its own reason
    bad_desc = _desc(de, 32, 3, 5, 60, 4, 1, 1, 0)
    assert L.dip_plan_workspace_bytes_opts(ctypes.byref(bad_desc), 512, 512, ctypes.byref(de.PlanOpts(de.PAD_ZERO))) == 0
    assert b"128" in L.dip_last_error()


def test_plan_rejects_unknown_pad_before_touching_the_device():
    import dip_engine as de
    with pytest.raises(ValueError, match="pad"):
        de.Plan(32, 3, 5, 128, 4, True, 64, 96, pad="replication")
