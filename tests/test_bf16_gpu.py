"""Precision mode 'bf16' (BASELINE.json configs[2]: "super-resolution x4 ... bf16") on the GPU.

What bf16 means here (DESIGN.md section 3, include/dip.h DIP_PRECISION_BF16): the wide convolutions run as wgmma
MMAs on bf16 operands -- their input, their weight and the incoming gradient are rounded to bf16 where the tensor-core
kernels read them -- with fp32 accumulation; master weights, biases, BatchNorm, activations, up-sampling, the skinny skip
convs, the head, the loss and Adam stay fp32.  The reference has no bf16 path; the checker is

  (a) layer-local, exact-level: every tensor-core convolution (forward, input gradient, weight gradient) against torch-CPU
      fp64 applied to the bf16 operands the engine itself read; the bf16 twins against the fp32 tensors they shadow;
  (b) whole network against the oracle evaluating exactly that definition on the CPU (`with O.operand_rounding('bf16')`), to
      the floor that definition has (the same oracle in fp32 vs fp64: rounding-boundary flips, see below);
  (c) the exact-fp32 oracle, against which the engine's bf16 error must not exceed the error of the reference's graph run by
      stock torch-CUDA under torch.autocast(bfloat16) (comparator only; it also rounds conv OUTPUTS to bf16, so it is the
      looser of the two).
"""
import numpy as np
import pytest
import torch

from oracle import dip_oracle as O
from baseline_cases import load_case, oracle_step, rel

pytestmark = pytest.mark.gpu

# Layer-local checks are exact-level (only the fp32 accumulation order differs); whole-network comparisons are not: a bf16
# rounding turns any 1e-7 difference into a full-ulp (2^-8) difference of the elements that sit on a rounding boundary, the
# next layer's flips follow the now larger difference, and three convolutions later two correct implementations differ by
# ~2^-9 everywhere (the bf16-operand oracle evaluated in fp32 and in fp64 ends 2e-2 apart at the last activation).  The
# whole-network tier therefore measures that floor (oracle fp32 vs oracle fp64, same definition) and holds the engine to it.
LOCAL_TOL = 3e-5    # relative Frobenius error of one conv output / input gradient given the engine's own bf16 operands
WGRAD_TOL = 1e-4    # weight gradients: split-K partial sums added with fp32 atomics
LOSS_TOL = 2e-3


def dead(name):
    return (name.endswith(".b") and "_bn" not in name and not name.startswith("head")) or name.endswith("cat_bn.b")


def make_plan(cfg, params, H, W):
    import dip_engine as de
    plan = de.Plan(cfg.in_channels, cfg.out_channels, cfg.num_scales, cfg.channels, cfg.skip_channels, cfg.upsample_mode == "bilinear", H, W,
                   precision=de.PRECISION_BF16, downsample_mode=cfg.downsample_mode)
    dparams = [p.detach().cuda().contiguous() for p in params]
    dgrads = [torch.zeros_like(p) for p in dparams]
    plan.bind(dparams, dgrads)
    return plan, dparams, dgrads


def chw(x_hwc):
    return x_hwc.permute(2, 0, 1).double().cpu()


def check_layers(tag, cfg, plan, params, dgrads):
    """Every tensor-core convolution of the step, forward / input gradient / weight gradient, against torch-CPU fp64 applied
    to the operands the engine itself read (its bf16 twins, plan.buffer('...16')), plus the twins against the fp32 tensors
    they shadow.  Engine channel order of the concat is [up | skip], torch's [skip | up]: roll by skip_channels."""
    import torch.nn.functional as F
    names = [n for n, _ in O.param_layout(cfg)]
    P = {n: p.detach().bfloat16().double() for n, p in zip(names, params)}     # weights as the kernels read them
    B = {n: p.detach().double() for n, p in zip(names, params)}
    G = {n: g.double().cpu() for n, g in zip(names, dgrads)}
    L = cfg.num_scales
    avg = cfg.downsample_mode == "avg"
    worst = {"fprop": ("", 0.0), "dgrad": ("", 0.0), "wgrad": ("", 0.0)}

    def upd(kind, key, got, ref):
        e = rel(got, ref)
        worst[kind] = max(worst[kind], (key, e), key=lambda t: t[1])

    for l in range(L):
        pf = "L%d." % l
        cs = cfg.ns(l)
        nd, nu, cc = cfg.nd(l), cfg.nu(l), cfg.cu(l) + cs
        pin = chw(plan.buffer(pf + "Pin16"))
        cin = P[pf + "d1.w"].shape[1]
        pin = pin[:cin]
        x_d2, x_up, x_11 = chw(plan.buffer(pf + "P_d1_16")), chw(plan.buffer(pf + "P_cat16")), chw(plan.buffer(pf + "A_u16"))
        x_up_t = torch.roll(x_up, cs, 0)
        # twins shadow the fp32 tensors exactly where those are kept
        assert torch.equal(plan.buffer(pf + "P_cat16"), plan.buffer(pf + "P_cat").bfloat16()), pf + "P_cat16"
        if l == 0 or cs == 4:
            assert torch.equal(plan.buffer(pf + "Pin16")[:, :, :cin], plan.buffer(pf + "Pin")[:, :, :cin].bfloat16()), pf + "Pin16"
        # forward
        if avg:   # stride-1 conv + AvgPool2d(2, 2) (models/common.py:101-105)
            upd("fprop", pf + "raw_d1", chw(plan.buffer(pf + "raw_d1")),
                F.avg_pool2d(F.conv2d(pin[None], P[pf + "d1.w"], B[pf + "d1.b"]), 2, 2)[0])
        else:
            upd("fprop", pf + "raw_d1", chw(plan.buffer(pf + "raw_d1")), F.conv2d(pin[None], P[pf + "d1.w"], B[pf + "d1.b"], stride=2)[0])
        upd("fprop", pf + "raw_d2", chw(plan.buffer(pf + "raw_d2")), F.conv2d(x_d2[None], P[pf + "d2.w"], B[pf + "d2.b"])[0])
        upd("fprop", pf + "raw_u", chw(plan.buffer(pf + "raw_u")), F.conv2d(x_up_t[None], P[pf + "up.w"], B[pf + "up.b"])[0])
        upd("fprop", pf + "raw_v", chw(plan.buffer(pf + "raw_v")), F.conv2d(x_11[None], P[pf + "c11.w"], B[pf + "c11.b"])[0])
        if cs == 128:
            upd("fprop", pf + "raw_s", chw(plan.buffer(pf + "raw_s")),
                F.conv2d(pin[None, :, 1:-1, 1:-1], P[pf + "skip.w"], B[pf + "skip.b"])[0])
        # the dropped fp32 tensors: the twin must be bf16(lrelu(bn(raw))) (+ reflection pad) up to rounding flips
        for raw_key, twin, pad in ((pf + "raw_d1", x_d2, 1), (pf + "raw_u", x_11, 0)):
            raw = chw(plan.buffer(raw_key)).float()
            g_, b_ = (params[names.index(pf + ("d1_bn" if pad else "up_bn") + s_)].detach() for s_ in (".g", ".b"))
            y = F.leaky_relu(F.batch_norm(raw[None], None, None, g_, b_, training=True, eps=1e-5), 0.2)
            if pad:
                y = F.pad(y, (1, 1, 1, 1), mode="reflect")
            yb = y[0].bfloat16().double()
            diff = (twin - yb).abs()
            # (an output next to zero is the difference of two O(1) terms: its own rounding error is absolute, ~1e-6; the
            # BatchNorm coefficients differ by ~1e-6 relative between torch's fp32 statistics and the engine's fp64 ones, so
            # about 1e-6 / 2^-8 ~ 1e-3 of the elements sit on the other side of a rounding boundary: measured 2e-4 .. 2.4e-3)
            assert (diff > 0).sum().item() <= 1e-2 * diff.numel() + 8 and (diff <= 2.0 ** -7 * yb.abs() + 1e-5).all(), raw_key
        # backward: dY twins -> input gradients and weight gradients
        dy_v, dy_u = chw(plan.buffer(pf + "dRaw_v16")), chw(plan.buffer(pf + "dRaw_u16"))
        dy_d2 = chw(plan.buffer(pf + "dRaw_d2_16"))
        if avg:   # the conv's dY = pooling adjoint of the (fp32) pooled gradient, rounded to bf16 where the kernels read it
            dy_d1 = (0.25 * plan.buffer(pf + "dRaw_d1")).bfloat16().permute(2, 0, 1).double().cpu()
            dy_d1 = dy_d1.repeat_interleave(2, 1).repeat_interleave(2, 2)
        else:
            dy_d1 = chw(plan.buffer(pf + "dRaw_d1_16"))
        upd("dgrad", pf + "dA_u", chw(plan.buffer(pf + "dA_u")), F.conv_transpose2d(dy_v[None], P[pf + "c11.w"])[0])
        upd("dgrad", pf + "dP_cat", chw(plan.buffer(pf + "dP_cat")), torch.roll(F.conv_transpose2d(dy_u[None], P[pf + "up.w"])[0], -cs, 0))
        upd("dgrad", pf + "dP_d1", chw(plan.buffer(pf + "dP_d1")), F.conv_transpose2d(dy_d2[None], P[pf + "d2.w"])[0])
        if l > 0 and avg:
            upd("dgrad", pf + "dPin", chw(plan.buffer(pf + "dPin")), F.conv_transpose2d(dy_d1[None], P[pf + "d1.w"])[0])
        elif l > 0:
            got = chw(plan.buffer(pf + "dPin"))
            ref = F.conv_transpose2d(dy_d1[None], P[pf + "d1.w"], stride=2)[0]
            upd("dgrad", pf + "dPin", got[:, :-1, :-1], ref)
            assert got[:, -1, :].abs().max() == 0 and got[:, :, -1].abs().max() == 0
        wg = torch.nn.grad.conv2d_weight
        upd("wgrad", pf + "c11.w", G[pf + "c11.w"], wg(x_11[None], (nu, nu, 1, 1), dy_v[None]))
        upd("wgrad", pf + "up.w", G[pf + "up.w"], wg(x_up_t[None], (nu, cc, 3, 3), dy_u[None]))
        upd("wgrad", pf + "d2.w", G[pf + "d2.w"], wg(x_d2[None], (nd, nd, 3, 3), dy_d2[None]))
        upd("wgrad", pf + "d1.w", G[pf + "d1.w"], wg(pin[None], (nd, cin, 3, 3), dy_d1[None], stride=1 if avg else 2)[:, :, :3, :3])
        if cs == 128:
            dy_s = chw(plan.buffer(pf + "dRaw_s16"))
            upd("wgrad", pf + "skip.w", G[pf + "skip.w"], wg(pin[None, :, 1:-1, 1:-1], (128, cin, 1, 1), dy_s[None]))
    print("\n[bf16 %s] layer-local worst relative errors: fprop %s %.1e | dgrad %s %.1e | wgrad %s %.1e" % (
        tag, worst["fprop"][0], worst["fprop"][1], worst["dgrad"][0], worst["dgrad"][1], worst["wgrad"][0], worst["wgrad"][1]))
    assert worst["fprop"][1] < LOCAL_TOL, worst["fprop"]
    assert worst["dgrad"][1] < LOCAL_TOL, worst["dgrad"]
    assert worst["wgrad"][1] < WGRAD_TOL, worst["wgrad"]


@pytest.mark.parametrize("kind", ["snail", "restoration_kate"])
def test_bf16_layers_per_scale_widths(kind):
    """The bf16 kernels on per-scale widths (K blocks with 8 / 16 / 32 valid channels of 64, wgmma N = 32 .. 128) and, for
    restoration.ipynb's kate network, the stride-1 first down conv behind downsample_mode='avg': layer-local, exact-level."""
    if kind == "snail":      # denoising.ipynb c8:13-23
        cfg = O.SkipConfig(in_channels=3, channels=[8, 16, 32, 64, 128], skip_channels=[0, 0, 0, 4, 4])
    else:                    # restoration.ipynb c7:28-36
        cfg = O.SkipConfig(in_channels=32, channels=[16, 32, 64, 128, 128], skip_channels=[0, 0, 0, 0, 0])
        cfg.downsample_mode = "avg"
    H, W = 64, 96
    params = O.init_params(cfg, seed=0)
    z0 = O.get_noise(cfg.in_channels, (H, W), seed=1)
    target = torch.rand(1, 3, H, W, generator=torch.Generator().manual_seed(2))
    plan, dparams, dgrads = make_plan(cfg, params, H, W)
    out = plan.forward(z0.cuda())
    plan.backward((2.0 * (out - target.cuda()) / out.numel()).contiguous())
    torch.cuda.synchronize()
    check_layers(kind, cfg, plan, params, dgrads)
    # and the whole step lands where the bf16-operand oracle does (floor-level agreement, see above)
    with O.operand_rounding("bf16"):
        ref = O.skip_forward(params, z0, cfg).detach()
    assert (out.cpu() - ref).abs().max().item() < 0.1


def net_errors(cfg, raw_get, out, grads, tape_ref, out_ref, grads_ref, raws):
    worst_raw = 0.0
    for l in range(cfg.num_scales):
        for nm in raws:
            key = "L%d.%s" % (l, nm)
            worst_raw = max(worst_raw, rel(raw_get(key), tape_ref[key][0].permute(1, 2, 0)))
    e_out = (out.double().cpu() - out_ref.double()).abs().max().item()
    names = [n for n, _ in O.param_layout(cfg)]
    gmax = max(x.norm().item() for x in grads_ref)
    ge = [rel(gd, gr) for name, gd, gr in zip(names, grads, grads_ref) if not dead(name) and gr.norm().item() >= 1e-4 * gmax]
    return worst_raw, e_out, float(np.median(ge)), float(max(ge))


def emulated_step(cfg, params, z, target, dtype):
    p = [x.detach().to(dtype).requires_grad_(True) for x in params]
    tape = {}
    with O.operand_rounding("bf16"):
        out = O.skip_forward(p, z.to(dtype), cfg, tape=tape)
        loss = O.mse_loss(out, target.to(dtype), None)
        grads = torch.autograd.grad(loss, p)
    return {k: v.detach() for k, v in tape.items() if "raw" in k}, out.detach(), loss.item(), grads


@pytest.mark.parametrize("shape_mode", [(64, 64, "bilinear", 4), (96, 64, "nearest", 4), (64, 96, "nearest", 128),
                                        (128, 64, "bilinear", 128), (64, 96, "nearest", 0), (128, 192, "bilinear", 4)])
def test_bf16_step_vs_bf16_operand_oracle(shape_mode):
    H, W, mode, cs = shape_mode
    cfg = O.SkipConfig(upsample_mode=mode, skip_channels=cs)
    params = O.init_params(cfg, seed=0)
    z0 = O.get_noise(32, (H, W), seed=1)
    target = torch.rand(1, 3, H, W, generator=torch.Generator().manual_seed(2))
    raws = ("raw_s", "raw_d1", "raw_d2", "raw_u", "raw_v")[0 if cs else 1:]
    t32, o32, l32, g32 = emulated_step(cfg, params, z0, target, torch.float32)
    t64, o64, l64, g64 = emulated_step(cfg, params, z0, target, torch.float64)
    floor = net_errors(cfg, lambda k: t32[k][0].permute(1, 2, 0), o32, g32, t64, o64, g64, raws)
    plan, dparams, dgrads = make_plan(cfg, params, H, W)
    out = plan.forward(z0.cuda())
    dout = (2.0 * (out - target.cuda()) / out.numel()).contiguous()
    plan.backward(dout)
    torch.cuda.synchronize()
    tag = "%dx%d %s cs=%d" % (H, W, mode, cs)
    check_layers(tag, cfg, plan, params, dgrads)
    mine = net_errors(cfg, plan.buffer, out, dgrads, t64, o64, g64, raws)
    print("[bf16 %s] whole network vs the bf16-operand oracle (fp64): worst pre-BN activation %.2e (floor %.2e) | output max abs "
          "%.2e (%.2e) | gradient error median %.3f (%.3f), worst %.3f (%.3f)" % (
              tag, mine[0], floor[0], mine[1], floor[1], mine[2], floor[2], mine[3], floor[3]))
    # (the floor is one sample of a chaotic quantity: measured engine / floor ratios 0.8 .. 2.2 over these shapes)
    assert mine[0] < 3.0 * floor[0] + 2e-3 and mine[1] < 3.0 * floor[1] + 2e-3, (mine, floor)
    assert mine[2] < 2.0 * floor[2] + 0.02, (mine, floor)


def engine_sr_step(c):
    """one closure step of the super-resolution configuration on the engine in bf16 (C ABI: forward, Lanczos operator, MSE,
    the operator's adjoint, backward)"""
    import dip_engine as de
    cfg, H, W = c["cfg"], c["H"], c["W"]
    plan, dparams, dgrads = make_plan(cfg, c["params"], H, W)
    out = plan.forward(c["z0"].cuda(), noise=c["noise"].cuda(), sigma=c["sigma"])
    L = de.lib()
    loss = torch.zeros(1, dtype=torch.float64, device="cuda")
    target = c["target"].cuda().contiguous()
    kern, f, pad = c["down"]
    kern = kern.cuda().contiguous()
    lr = de.lanczos_down_fwd(out, kern, f, pad)
    dlr = torch.empty_like(lr)
    de.check(L.dip_loss_mse(lr.data_ptr(), target.data_ptr(), None, 3, lr.shape[2] * lr.shape[3], loss.data_ptr(),
                            dlr.data_ptr(), None))
    dout = de.lanczos_down_bwd(dlr, kern, f, pad, H, W)
    plan.backward(dout)
    torch.cuda.synchronize()
    return plan, out, loss.item(), dgrads


def autocast_bf16_grads(c):
    """comparator: the reference's graph on stock torch-CUDA under autocast(bfloat16)"""
    pc = [p.detach().cuda().requires_grad_(True) for p in c["params"]]
    z = (c["z0"] + c["noise"] * c["sigma"]).cuda()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out = O.skip_forward(pc, z, c["cfg"])
    out = out.float()
    kern, f, pad = c["down"]
    x = torch.nn.functional.pad(out, (pad,) * 4, mode="replicate")
    w = torch.zeros(3, 3, *kern.shape, device="cuda")
    for i in range(3):
        w[i, i] = kern.cuda()
    o = torch.nn.functional.conv2d(x, w, stride=f)
    loss = O.mse_loss(o, c["target"].cuda(), None)
    return [x.detach().float().cpu() for x in torch.autograd.grad(loss, pc)], out.detach().cpu()


@pytest.mark.parametrize("kind", ["sr_zebra", "sr1024"])
def test_bf16_sr_step_at_baseline_shape(kind):
    """BASELINE config 3 (zebra 384x576 -> 96x144, and the 1024^2 -> 256^2 shape of BASELINE's wording), one step in bf16:
    (a) every convolution layer-locally, (c) the whole step against the exact-fp32 oracle, error no larger than that of the
    reference's graph under torch.autocast(bfloat16) on the same GPU."""
    c = load_case(kind)
    cfg = c["cfg"]
    plan, out, loss, dgrads = engine_sr_step(c)
    check_layers(kind, cfg, plan, c["params"], dgrads)
    del plan
    ce = oracle_step(kind)
    assert abs(loss - ce["loss"]) < LOSS_TOL, (loss, ce["loss"])
    gc, out_c = autocast_bf16_grads(c)
    names = [n for n, _ in O.param_layout(cfg)]
    gmax = max(x.norm().item() for x in ce["grads"])
    e_ours, e_auto = [], []
    for name, gd, ga, gr in zip(names, dgrads, gc, ce["grads"]):
        if dead(name) or gr.norm().item() < 1e-4 * gmax:
            continue
        e_ours.append(rel(gd, gr))
        e_auto.append(rel(ga, gr))
    eo, ea = (out.cpu() - ce["out"]).abs().max().item(), (out_c - ce["out"]).abs().max().item()
    print("[bf16 %s] vs the exact-fp32 oracle: output max abs engine %.2e / autocast %.2e | gradient error median engine %.3f / "
          "autocast %.3f, worst engine %.3f / autocast %.3f | loss %.6f (fp32 oracle %.6f)" % (
              kind, eo, ea, np.median(e_ours), np.median(e_auto), max(e_ours), max(e_auto), loss, ce["loss"]))
    assert eo < 1.5 * ea + 2e-3, (eo, ea)
    assert np.median(e_ours) < 1.2 * np.median(e_auto) + 0.01, (np.median(e_ours), np.median(e_auto))
    torch.cuda.empty_cache()


def test_bf16_module_api_runs_and_tracks_tf32():
    """net.precision = 'bf16' through the notebook-facing modules (get_net / Downsampler / optimize): 300 iterations of the
    super-resolution closure at 256x384 -> 64x96; the loss must fall like the tf32 run's from the same initial state."""
    import models
    from utils import common_utils as cu
    dtype = torch.cuda.FloatTensor
    H, W, iters = 256, 384, 300
    g = torch.Generator().manual_seed(5)
    hr = torch.nn.functional.interpolate(torch.rand(1, 3, H // 8, W // 8, generator=g), size=(H, W), mode="bicubic",
                                         align_corners=False).clamp(0, 1)
    finals = {}
    for prec in ("tf32", "bf16"):
        torch.manual_seed(0)
        net = models.get_net(32, "skip", "reflection", skip_n33d=128, skip_n33u=128, skip_n11=4, num_scales=5,
                             upsample_mode="bilinear").type(dtype)
        net.precision = prec
        down = models.Downsampler(n_planes=3, factor=4, kernel_type="lanczos2", phase=0.5, preserve_size=True).type(dtype)
        with torch.no_grad():
            lr = down(hr.type(dtype)).detach()
        torch.manual_seed(1)
        z0 = cu.get_noise(32, "noise", (H, W)).type(dtype).detach()
        gn = torch.Generator(device="cuda").manual_seed(9)
        mse = torch.nn.MSELoss().type(dtype)
        losses, psnr = [], []

        def closure():
            out_hr = net(z0 + torch.randn(z0.shape, generator=gn, device="cuda") * 0.03)
            loss = mse(down(out_hr), lr)
            loss.backward()
            losses.append(loss.item())
            psnr.append(O.psnr(hr.numpy()[0], out_hr.detach().cpu().numpy()[0]))
            return loss

        cu.optimize("adam", cu.get_params("net", net, z0), closure, 0.01, iters)
        finals[prec] = (losses[0], float(np.mean(losses[-20:])), float(np.mean(psnr[-20:])))
    print("\n[bf16 module API] loss first / tail-20 mean / PSNR_HR tail-20 mean: tf32 %s | bf16 %s" % (finals["tf32"], finals["bf16"]))
    assert abs(finals["bf16"][0] - finals["tf32"][0]) < 5e-3
    assert finals["bf16"][1] < 0.2 * finals["bf16"][0]                      # it optimises
    assert abs(finals["bf16"][2] - finals["tf32"][2]) < 1.0                 # and ends where the tf32 run ends (dB)
