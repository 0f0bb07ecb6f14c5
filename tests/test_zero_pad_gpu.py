"""Zero padding on the engine (H100): every stage of one forward + backward against its fp64 reference at the engine's
own inputs (tests/stage_ref.py under pad_refs.padding, the tolerances of tests/test_stages_gpu.py, every registered buffer
NaN-filled first), exact-zero halos of every conv input and its bf16 twin, and the notebook-facing API against fixtures
of the unmodified reference (tests/golden/make_zero_pad.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import dip_oracle as O
import pad_refs as PR
import stage_ref as SR
import test_stages_gpu as TS
from test_zero_pad_cpu import CASES as GOLD_CASES, GOLD, build_skip, setup

pytestmark = pytest.mark.gpu
MODES = ["fp32", "tf32", "bf16"]
HALO_BUFFERS = ["Pin", "P_d1", "P_d2", "P_cat", "Pin16", "P_d1_16", "P_d2_16", "P_cat16"]


def cfg_of(kind):
    if kind == "skipdefault":   # models.skip(32, 3): widths [16, 32, 64, 128, 128], skips 4, nearest
        cfg = O.SkipConfig(upsample_mode="nearest", channels=[16, 32, 64, 128, 128], skip_channels=[4] * 5)
    else:
        cfg = TS.cfg_of(kind)
    cfg.pad = "zero"
    return cfg


def make_plan(cfg, H, W, mode, input_grad=False):
    import dip_engine as de
    prec = {"fp32": de.PRECISION_FP32, "tf32": de.PRECISION_TF32, "bf16": de.PRECISION_BF16}[mode]
    bil = cfg.upsample_mode == "bilinear" if isinstance(cfg.upsample_mode, str) else [m == "bilinear" for m in cfg.upsample_mode]
    L = cfg.num_scales
    per_scale = isinstance(cfg.channels, (list, tuple)) or isinstance(cfg.skip_channels, (list, tuple))
    ch = [cfg.nd(l) for l in range(L)] if per_scale else cfg.channels
    sk = [cfg.ns(l) for l in range(L)] if per_scale else cfg.skip_channels
    return de.Plan(cfg.in_channels, cfg.out_channels, L, ch, sk, bil, H, W, precision=prec, need_sigmoid=cfg.need_sigmoid,
                   input_grad=input_grad, downsample_mode=cfg.downsample_mode, pad=cfg.pad)


def check_halos(cfg, mode, plan):
    """the halo ring of every padded conv input (and of its bf16 twin) holds exact zeros"""
    bad, n = [], 0
    for l in range(cfg.num_scales):
        for b in HALO_BUFFERS:
            name = "L%d.%s" % (l, b)
            if b.startswith("P_d2") and l == cfg.num_scales - 1:
                continue   # the deepest level's P_d2 is plain (no conv reads it padded)
            if mode == "bf16" and not b.endswith("16") and (
                    TS.fp32_dropped(cfg, name) or (b == "Pin" and l > 0 and TS.fp32_dropped(cfg, "L%d.P_d2" % (l - 1)))):
                continue   # never written in bf16 mode (its twin is checked; a level's Pin is the P_d2 of the level above)
            v = TS.buffer_view(plan, name)
            if v is None or not v.numel():
                continue
            v = v.float()
            ring = torch.cat([v[0].flatten(), v[-1].flatten(), v[:, 0].flatten(), v[:, -1].flatten()])
            n += 1
            if not torch.equal(ring, torch.zeros_like(ring)):
                bad.append("%s: %d non-zero halo cells" % (name, (ring != 0).sum().item()))
    assert n > 0
    assert not bad, "[%s] " % mode + "; ".join(bad)


def run_direct(cfg, H, W, mode, input_grad=False, seed=0):
    params = TS.params_for(cfg, seed)
    g = torch.Generator().manual_seed(seed + 1)
    z = torch.rand(1, cfg.in_channels, H, W, generator=g).cuda()
    target = torch.rand(1, cfg.out_channels, H, W, generator=g).cuda()
    plan = make_plan(cfg, H, W, mode, input_grad)
    dparams = [p.cuda().contiguous() for p in params]
    dgrads = [torch.zeros_like(p) for p in dparams]
    plan.bind(dparams, dgrads)
    TS.fill_nan(plan, cfg.num_scales)
    out = plan.forward(z)
    dout = (2.0 * (out - target) / out.numel()).contiguous()
    plan.backward(dout)
    dz = plan.input_grad() if input_grad else None
    torch.cuda.synchronize()
    check_halos(cfg, mode, plan)
    refs = SR.Refs()
    src = plan.buffer if mode != "bf16" else (lambda n: TS.buffer_view(plan, n) if n.endswith("16") else plan.buffer(n))
    PR.stage_forward(cfg, dparams, lambda n: out[0] if n == "out" else src(n), mode, refs, z=z)
    PR.stage_backward(cfg, dparams, lambda n: out[0] if n == "out" else src(n), mode, refs, dout[0], input_grad=input_grad)
    TS.check("zero-pad %s %dx%d" % (TS.cfg_tag(cfg), H, W), cfg, mode, plan, refs, dgrads, out, dz)
    return plan, out, dgrads


CASES = [("cs4", 64, 96, False), ("skipdefault", 64, 96, False), ("cs128", 96, 64, False), ("cs0", 64, 96, False),
         ("kate", 96, 64, False), ("ingrad", 64, 96, True)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", CASES, ids=["%s_%dx%d" % c[:3] for c in CASES])
def test_every_stage_zero_pad(case, mode):
    kind, H, W, input_grad = case
    run_direct(cfg_of(kind), H, W, mode, input_grad)
    TS.print_table()


def run_runner(cfg, H, W, mode, task):
    """one iteration of the device runner (fused noise + zero-padded input) at lr = 0, every stage checked"""
    import dip_engine as de
    params = TS.params_for(cfg, 3)
    g = torch.Generator().manual_seed(5)
    z0 = torch.rand(1, cfg.in_channels, H, W, generator=g).cuda()
    plan = make_plan(cfg, H, W, mode)
    mask = down = None
    if task == "sr":
        kern = O.down_kernel(4, "lanczos2", 0.5)
        down = (torch.from_numpy(kern).double(), 4, O.down_pad(kern.shape[0], 4))
        plan.set_downsampler(torch.from_numpy(kern).float(), 4, down[2])
        th, tw = de.down_out_size(H, kern.shape[0], 4, down[2]), de.down_out_size(W, kern.shape[0], 4, down[2])
    else:
        th, tw = H, W
    target = torch.rand(1, cfg.out_channels, th, tw, generator=g).cuda()
    if task == "inpaint":
        mask = (torch.rand(1, 1, H, W, generator=g) > 0.3).float().cuda()
    dparams = [p.cuda().contiguous() for p in params]
    dgrads = [torch.zeros_like(p) for p in dparams]
    plan.bind(dparams, dgrads)
    for p, gb in zip(dparams, dgrads):
        p.grad = gb
    adam = de.FusedAdam(dparams, lr=0.0)
    adam._bind(dgrads)
    before = [p.clone() for p in dparams]
    TS.fill_nan(plan, cfg.num_scales)
    out = torch.empty(1, cfg.out_channels, H, W, device="cuda")
    de.run_iterations(plan, adam, z0, target, mask, 1. / 30, 7, 1, 0.0, out=out)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(before, dparams))
    check_halos(cfg, mode, plan)
    o = out.double().cpu().requires_grad_(True)
    lo = o if down is None else O.downsample(o, *down)
    loss = O.mse_loss(lo, target.double().cpu(), None if mask is None else mask.double().cpu())
    dout = torch.autograd.grad(loss, o)[0].cuda()
    src = plan.buffer if mode != "bf16" else (lambda n: TS.buffer_view(plan, n) if n.endswith("16") else plan.buffer(n))
    rd = lambda n: out[0] if n == "out" else src(n)   # noqa: E731
    refs = SR.Refs()
    PR.stage_forward(cfg, dparams, rd, mode, refs)
    PR.stage_backward(cfg, dparams, rd, mode, refs, dout[0])
    TS.check("zero-pad runner %s %s %dx%d" % (task, TS.cfg_tag(cfg), H, W), cfg, mode, plan, refs, dgrads, out)


@pytest.mark.parametrize("task,kind,H,W,mode", [("denoise", "cs4", 128, 128, "tf32"), ("inpaint", "cs128", 128, 192, "tf32"),
                                                 ("sr", "cs4", 256, 256, "tf32"), ("sr", "cs4", 256, 256, "bf16")])
def test_every_stage_runner_zero_pad(task, kind, H, W, mode):
    run_runner(cfg_of(kind), H, W, mode, task)
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
