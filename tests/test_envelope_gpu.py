"""The envelope table (tests/envelope_cases.py) on the engine (H100): 1 to 8 scales, every width class, unequal down / up
widths, input depths 1 to 100, 1 to 4 outputs.  Every stage of one forward + backward is checked against its fp64
reference at the engine's own inputs, in fp32, tf32 and bf16, with every registered buffer NaN-filled first (the
machinery and tolerances of tests/test_stages_gpu.py, unchanged); rows marked zero_pad run again with pad='zero' and
exact-zero halos.  The device runner runs at lr = 0 on three rows (the split-noise path at W % 4 = 2, masked inpainting,
x4 super-resolution), and three rows go through models.skip against the oracle's fp64 autograd."""
import torch
import torch.nn.functional as F
import pytest

from oracle import dip_oracle as O
import envelope_cases as E
import pad_refs as PR
import stage_ref as SR
import test_stages_gpu as TS
from test_zero_pad_gpu import check_halos

pytestmark = pytest.mark.gpu
MODES = ["fp32", "tf32", "bf16"]


def make_plan(cfg, H, W, mode, input_grad=False):
    """dip_engine.Plan of an oracle SkipConfig with per-scale down / up / skip widths, up modes and padding"""
    import dip_engine as de
    prec = {"fp32": de.PRECISION_FP32, "tf32": de.PRECISION_TF32, "bf16": de.PRECISION_BF16}[mode]
    L = cfg.num_scales
    return de.Plan(cfg.in_channels, cfg.out_channels, L, [cfg.nd(l) for l in range(L)], [cfg.ns(l) for l in range(L)],
                   [SR._up_mode(cfg, l) for l in range(L)], H, W, precision=prec, need_sigmoid=cfg.need_sigmoid,
                   input_grad=input_grad, channels_up=[cfg.nu(l) for l in range(L)], downsample_mode=cfg.downsample_mode,
                   pad=cfg.pad)


def engine_src(plan, mode, out):
    src = plan.buffer if mode != "bf16" else (lambda n: TS.buffer_view(plan, n) if n.endswith("16") else plan.buffer(n))
    return lambda n: out[0] if n == "out" else src(n)


def run_direct(row, pad, mode, seed=0):
    cfg = E.cfg_of(row, pad)
    H, W = row.H, row.W
    params = TS.params_for(cfg, seed)
    g = torch.Generator().manual_seed(seed + 1)
    z = torch.rand(1, cfg.in_channels, H, W, generator=g).cuda()
    target = torch.rand(1, cfg.out_channels, H, W, generator=g).cuda()
    plan = make_plan(cfg, H, W, mode, row.input_grad)
    dparams = [p.cuda().contiguous() for p in params]
    dgrads = [torch.zeros_like(p) for p in dparams]
    plan.bind(dparams, dgrads)
    TS.fill_nan(plan, cfg.num_scales)
    out = plan.forward(z)
    dout = (2.0 * (out - target) / out.numel()).contiguous()
    plan.backward(dout)
    dz = plan.input_grad() if row.input_grad else None
    torch.cuda.synchronize()
    if pad == "zero":
        check_halos(cfg, mode, plan)
    refs = SR.Refs()
    rd = engine_src(plan, mode, out)
    PR.stage_forward(cfg, dparams, rd, mode, refs, z=z)
    PR.stage_backward(cfg, dparams, rd, mode, refs, dout[0], input_grad=row.input_grad)
    TS.check("envelope %s pad=%s %dx%d" % (row.id, pad, H, W), cfg, mode, plan, refs, dgrads, out, dz)


STAGE_CASES = [(r.id, pad) for r in E.ROWS for pad in E.pads_of(r)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("rid,pad", STAGE_CASES, ids=["%s_%s" % c for c in STAGE_CASES])
def test_every_stage_envelope(rid, pad, mode):
    run_direct(E.BY_ID[rid], pad, mode)
    TS.print_table()


def run_runner(row, H, W, mode, task):
    """one iteration of the device runner at lr = 0 (as test_stages_gpu.run_runner), every stage checked; the level-0
    padded input it leaves is pad(dip_noise_perturb(offset 0)) bit for bit, with exact zeros in the stored depth's
    channels after the real ones"""
    import dip_engine as de
    cfg = E.cfg_of(row)
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
    sigma, seed = 1. / 30, 7
    de.run_iterations(plan, adam, z0, target, mask, sigma, seed, 1, 0.0, out=out)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(before, dparams))

    zn = torch.empty_like(z0)
    de.check(de.lib().dip_noise_perturb(z0.data_ptr(), zn.data_ptr(), sigma, seed, 0, z0.numel(), None))
    torch.cuda.synchronize()
    want = SR.reflect_pad(SR.hwc(zn.double()))
    pin = plan.buffer("L0.Pin")
    c = cfg.in_channels
    assert pin.shape[-1] == SR.stored_depth(cfg, 0)
    assert torch.equal(pin[..., c:], torch.zeros_like(pin[..., c:])), "stored-depth channels after the input's are not zero"
    assert torch.equal(pin[..., :c].double(), want), (pin[..., :c].double() - want).abs().max().item()

    o = out.double().cpu().requires_grad_(True)
    lo = o if down is None else O.downsample(o, *down)
    loss = O.mse_loss(lo, target.double().cpu(), None if mask is None else mask.double().cpu())
    dout = torch.autograd.grad(loss, o)[0].cuda()
    rd = engine_src(plan, mode, out)
    refs = SR.Refs()
    SR.forward(cfg, dparams, rd, mode, refs)
    SR.backward(cfg, dparams, rd, mode, refs, dout[0])
    TS.check("envelope runner %s %s %dx%d" % (task, row.id, H, W), cfg, mode, plan, refs, dgrads, out)


@pytest.mark.parametrize("task,rid,H,W,mode", [("denoise", "L1", 10, 14, "tf32"), ("denoise", "L1", 10, 14, "bf16"),
                                                ("inpaint", "L4", 32, 48, "tf32"), ("sr", "rev5", 128, 128, "bf16")])
def test_every_stage_envelope_runner(task, rid, H, W, mode):
    run_runner(E.BY_ID[rid], H, W, mode, task)
    TS.print_table()


@pytest.mark.parametrize("rid", [r.id for r in E.ROWS if r.module])
def test_models_skip_vs_oracle_fp32(rid):
    """models.skip(...) at the row's arguments, precision 'fp32', one forward + backward with dL/d(input): the spec ->
    Plan mapping, against the oracle's fp64 autograd at the bounds of test_variants.py's
    test_input_gradient_and_no_sigmoid_vs_oracle"""
    import models
    row = E.BY_ID[rid]
    cfg = E.cfg_of(row)
    params = O.init_params(cfg, seed=0, dtype=torch.float64)
    gen = torch.Generator().manual_seed(2)
    z0 = (torch.rand(1, row.in_ch, row.H, row.W, generator=gen, dtype=torch.float64) * 0.1).requires_grad_(True)
    target = torch.rand(1, row.out_ch, row.H, row.W, generator=gen, dtype=torch.float64)
    out_ref = O.skip_forward(params, z0, cfg)
    grads_ref = torch.autograd.grad(O.mse_loss(out_ref, target), [z0] + params)

    torch.manual_seed(0)
    net = models.skip(**E.skip_kwargs(row)).type(torch.cuda.FloatTensor)
    assert net._dip_spec is not None, net._dip_why
    net.precision = "fp32"
    zd = z0.detach().float().cuda().requires_grad_(True)
    out = net(zd)
    F.mse_loss(out, target.float().cuda()).backward()
    err = (out.detach().double().cpu() - out_ref.detach()).abs().max().item()
    assert err < 5e-4, err

    def rel(a, b):
        a = a.double().cpu()
        return ((a - b).norm() / (b.norm() + 1e-30)).item()
    assert zd.grad is not None and rel(zd.grad, grads_ref[0]) < 3e-2, rel(zd.grad, grads_ref[0])
    gmax = max(g.norm().item() for g in grads_ref[1:])
    names = [n for n, _ in O.param_layout(cfg)]
    for name, p, g in zip(names, net.parameters(), grads_ref[1:]):
        if g.norm().item() > 1e-4 * gmax:
            assert rel(p.grad, g) < 3e-2, (name, rel(p.grad, g))
