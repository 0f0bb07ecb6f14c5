"""Zero padding on the engine (H100): every stage of the zero-padded networks against the fp64 references, through the
harness of tests/test_stages_gpu.py (which also checks that every halo cell holds an exact zero), and the
notebook-facing API against fixtures of the unmodified reference (tests/golden/make_zero_pad.py)."""
import os

import numpy as np
import pytest
import torch

import envelope_cases as E
import test_stages_gpu as TS
from test_zero_pad_cpu import CASES as GOLD_CASES, GOLD, build_skip, setup

pytestmark = pytest.mark.gpu
MODES = ["fp32", "tf32", "bf16"]
CASES = [("cs4", 64, 96, False), ("skipdefault", 64, 96, False), ("cs128", 96, 64, False), ("cs0", 64, 96, False),
         ("kate", 96, 64, False), ("ingrad", 64, 96, True)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", CASES, ids=["%s_%dx%d" % c[:3] for c in CASES])
def test_every_stage_zero_pad(case, mode):
    kind, H, W, input_grad = case
    TS.run_direct(E.cfg_of(kind, "zero"), H, W, mode, input_grad)
    TS.print_table()


@pytest.mark.parametrize("task,kind,H,W,mode", [("denoise", "cs4", 128, 128, "tf32"), ("inpaint", "cs128", 128, 192, "tf32"),
                                                 ("sr", "cs4", 256, 256, "tf32"), ("sr", "cs4", 256, 256, "bf16")])
def test_every_stage_runner_zero_pad(task, kind, H, W, mode):
    TS.run_runner(E.cfg_of(kind, "zero"), H, W, mode, task)
    TS.print_table()


@pytest.mark.parametrize("prec", ["fp32", "tf32"])
@pytest.mark.parametrize("case", GOLD_CASES)
def test_engine_matches_reference_golden_zero_pad(case, prec):
    """One closure step through models.skip + optimize vs the reference's numbers (fp32 fixture), at the tiers of
    tests/test_variants.py"""
    import models
    from utils.common_utils import get_params, optimize
    g = np.load(os.path.join(GOLD, case + "_fp32.npz"))
    cfg, z0, target, mask, noises = setup(g, torch.float32)
    dtype = torch.cuda.FloatTensor
    torch.manual_seed(0)
    net = (models.skip(32, 3) if case.startswith("skipdefault") else build_skip(g)).type(dtype)
    assert net._dip_spec["pad"] == "zero"
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
    tol_out, tol_loss, tol_g = (1e-4, 1e-5, 3e-2) if prec == "fp32" else (2e-2, 1e-3, 0.25)
    assert np.abs(outs[0].cpu().numpy() - g["out0"]).max() < tol_out
    assert abs(losses[0] - float(g["losses"][0])) < tol_loss
    gnorm = np.array([p.grad.double().norm().item() for p in params])
    big = g["gnorm0"] > 1e-4 * g["gnorm0"].max()
    dev = np.abs(gnorm[big] / g["gnorm0"][big] - 1)
    assert (np.median(dev) if prec == "tf32" else dev.max()) < (0.1 if prec == "tf32" else tol_g), dev.max()

    def rel(a, b):
        a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double()
        return ((a - b).norm() / (b.norm() + 1e-30)).item()
    skips = [int(x) for x in g["skips"]]
    tol1 = 3e-2 if prec == "fp32" else (0.3 if skips[0] else 0.6)
    assert rel(params[0].grad, g["g_skip0_w"]) < tol1
    assert rel(params[4 if skips[0] else 0].grad, g["g_d1_0_w"]) < tol1
    optimize("adam", params, closure, float(g["lr"]), 2)
    assert np.isfinite(losses).all() and abs(losses[1] - float(g["losses"][1])) < 2e-2
