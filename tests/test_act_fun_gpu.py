"""Activations other than LeakyReLU on the engine (H100): every stage of the networks with each activation against the
fp64 references, through the harness of tests/test_stages_gpu.py (which also checks that no element is excluded from
the backward checks), the notebook-facing API against fixtures of the unmodified reference (tests/golden/make_act_fun.py),
and LeakyReLU given explicitly = NULL options."""
import ctypes
import os

import numpy as np
import pytest
import torch

import envelope_cases as E
import test_stages_gpu as TS
from test_act_fun_cpu import CASES as GOLD_CASES, GOLD, build_net
from test_zero_pad_cpu import setup

pytestmark = pytest.mark.gpu
MODES = ["fp32", "tf32", "bf16"]
KINDS = ["Swish", "ELU", "none"]

NETS = {"cs4": (64, 96, False), "skipdefault": (64, 96, False), "cs128": (96, 64, False), "cs0": (64, 96, False),
        "kate": (96, 64, False), "snail": (64, 96, False), "ingrad": (64, 96, True)}
# every kind meets every network; cs4 and the skip() default network in all three modes, the others in one mode each,
# rotated so that every (kind, mode) pair occurs
ONE_MODE = {"cs128": ("tf32", "bf16", "fp32"), "cs0": ("bf16", "fp32", "tf32"), "kate": ("fp32", "tf32", "bf16"),
            "snail": ("tf32", "bf16", "fp32"), "ingrad": ("bf16", "fp32", "tf32")}
DIRECT = [(net, act, mode) for net in ("cs4", "skipdefault") for act in KINDS for mode in MODES] + \
         [(net, act, modes[i]) for net, modes in ONE_MODE.items() for i, act in enumerate(KINDS)]

PAD = {"skipdefault": "zero"}   # the skip() default network as models.skip builds it; the others pad by reflection


@pytest.mark.parametrize("net,act,mode", DIRECT, ids=["%s_%s_%s" % c for c in DIRECT])
def test_every_stage_act(net, act, mode):
    H, W, input_grad = NETS[net]
    TS.run_direct(E.cfg_of(net, PAD.get(net, "reflection"), act), H, W, mode, input_grad)
    TS.print_table()


@pytest.mark.parametrize("task,act,kind,H,W,mode", [("denoise", "Swish", "cs4", 128, 128, "tf32"),
                                                     ("inpaint", "ELU", "cs128", 128, 192, "tf32"),
                                                     ("sr", "none", "cs4", 256, 256, "tf32"),
                                                     ("sr", "none", "cs4", 256, 256, "bf16")])
def test_every_stage_runner_act(task, act, kind, H, W, mode):
    TS.run_runner(E.cfg_of(kind, PAD.get(kind, "reflection"), act), H, W, mode, task)
    TS.print_table()


def closure_run(case, prec, steps):
    """models.skip / get_net + optimize as the notebooks call them, on the fixture's inputs: (losses, outputs, params)"""
    from utils.common_utils import get_params, optimize
    g = np.load(os.path.join(GOLD, case + "_fp32.npz"))
    cfg, z0, target, mask, noises = setup(g, torch.float32)
    dtype = torch.cuda.FloatTensor
    torch.manual_seed(0)
    net = build_net(case, g).type(dtype)
    assert net._dip_spec["act_fun"] == str(g["act_fun"])
    net.precision = prec
    z0d, tgt = z0.type(dtype), target.type(dtype)
    md = mask.type(dtype) if mask is not None else None
    mse = torch.nn.MSELoss().type(dtype)
    it = iter(noises)
    losses, outs = [], []

    def closure():
        out = net(z0d + next(it).type(dtype) * float(g["sigma"]))
        loss = mse(out * md, tgt * md) if md is not None else mse(out, tgt)
        loss.backward()
        losses.append(loss.item())
        outs.append(out.detach())
        return loss

    params = get_params("net", net, z0d)
    optimize("adam", params, closure, float(g["lr"]), 1)
    grads = [p.grad.clone() for p in params]
    if steps > 1:
        optimize("adam", params, closure, float(g["lr"]), steps - 1)
    return g, losses, outs, grads


@pytest.mark.parametrize("prec", ["fp32", "tf32"])
@pytest.mark.parametrize("case", GOLD_CASES)
def test_engine_matches_reference_golden_act(case, prec):
    """One closure step through models.skip / get_net + optimize vs the reference's numbers (fp32 fixture), at the tiers
    of tests/test_zero_pad_gpu.py; then two more steps, finite and close"""
    g, losses, outs, grads = closure_run(case, prec, 3)
    tol_out, tol_loss, tol_g = (1e-4, 1e-5, 3e-2) if prec == "fp32" else (2e-2, 1e-3, 0.25)
    assert np.abs(outs[0].cpu().numpy() - g["out0"]).max() < tol_out
    assert abs(losses[0] - float(g["losses"][0])) < tol_loss
    gnorm = np.array([x.double().norm().item() for x in grads])
    big = g["gnorm0"] > 1e-4 * g["gnorm0"].max()
    dev = np.abs(gnorm[big] / g["gnorm0"][big] - 1)
    assert (np.median(dev) if prec == "tf32" else dev.max()) < (0.1 if prec == "tf32" else tol_g), dev.max()

    def rel(a, b):
        a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double()
        return ((a - b).norm() / (b.norm() + 1e-30)).item()
    skips = [int(x) for x in g["skips"]]
    tol1 = 3e-2 if prec == "fp32" else (0.3 if skips[0] else 0.6)
    assert rel(grads[0], g["g_skip0_w"]) < tol1
    assert rel(grads[4 if skips[0] else 0], g["g_d1_0_w"]) < tol1
    assert np.isfinite(losses).all() and abs(losses[1] - float(g["losses"][1])) < 2e-2


@pytest.mark.parametrize("case", GOLD_CASES)
def test_engine_runs_act_fixture_in_bf16(case):
    """precision 'bf16' on the same networks: one step finite and near the reference's fp32 output (the bound of smoke():
    bf16 conv operands against an fp32 network at 64 x 96, where the deepest BatchNorms see 4 x 6 pixels)"""
    g, losses, outs, grads = closure_run(case, "bf16", 1)
    assert all(torch.isfinite(x).all() for x in grads) and torch.isfinite(outs[0]).all()
    assert np.abs(outs[0].cpu().numpy() - g["out0"]).max() < 0.15
    assert abs(losses[0] - float(g["losses"][0])) < 5e-3


def _null_opts(plan):
    """re-create plan's handle through dip_plan_create, which passes NULL options"""
    import dip_engine as de
    L = de.lib()
    nbytes = L.dip_plan_workspace_bytes(ctypes.byref(plan.desc), plan.H, plan.W)
    assert nbytes > 0 and nbytes + 512 <= plan.workspace.numel()
    L.dip_plan_destroy(plan.h)
    base = (plan.workspace.data_ptr() + 255) // 256 * 256
    h = ctypes.c_void_p()
    with torch.cuda.device(plan.device):
        de.check(L.dip_plan_create(ctypes.byref(plan.desc), plan.H, plan.W, ctypes.c_void_p(base), nbytes, ctypes.byref(h)))
    plan.h = h
    plan._bound_key = None
    return plan


@pytest.mark.parametrize("mode", MODES)
def test_explicit_leaky_relu_equals_null_opts(mode):
    """act_fun = DIP_ACT_LEAKY_RELU given explicitly computes bitwise what a plan with NULL options computes (and Swish
    does not)"""
    import dip_engine as de
    cfg = E.cfg_of("cs4")
    H, W = 64, 96
    params = [p.cuda().contiguous() for p in TS.params_for(cfg, 0)]
    g = torch.Generator().manual_seed(1)
    z = torch.rand(1, cfg.in_channels, H, W, generator=g).cuda()
    target = torch.rand(1, cfg.out_channels, H, W, generator=g).cuda()
    results = {}
    for name in ("explicit", "null", "swish"):
        cfg.act_fun = "Swish" if name == "swish" else "LeakyReLU"
        plan = TS.make_plan(cfg, H, W, mode)
        if name == "explicit":
            assert (plan.opts.pad_mode, plan.opts.act_fun) == (de.PAD_REFLECTION, de.ACT_LEAKY_RELU)
        if name == "null":
            plan = _null_opts(plan)
        grads = [torch.zeros_like(p) for p in params]
        plan.bind(params, grads)
        out = plan.forward(z)
        plan.backward((2.0 * (out - target) / out.numel()).contiguous())
        torch.cuda.synchronize()
        results[name] = (out.clone(), [x.clone() for x in grads])
    (oa, ga), (ob, gb), (os_, gs) = results["explicit"], results["null"], results["swish"]
    assert torch.equal(oa, ob)
    assert all(torch.equal(a, b) for a, b in zip(ga, gb))
    assert not torch.equal(oa, os_) and not all(torch.equal(a, b) for a, b in zip(ga, gs))
