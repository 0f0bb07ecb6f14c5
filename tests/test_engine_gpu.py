"""P1/P2 tiers on the GPU: the CUDA engine (through the C ABI) vs the CPU oracle and the committed reference goldens.

Tolerances (SURVEY.md 7.4): fp32 mode is compared tightly (no TF32 rounding); tf32 mode = cuDNN's default fp32
behaviour, compared loosely.  Conv biases in front of a BatchNorm have mathematically-zero gradients (pure rounding
noise in the reference too) and are excluded from relative comparisons.
"""
import os

import numpy as np
import pytest
import torch

from oracle import dip_oracle as O

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

FWD_TOL = {"fp32": 1e-4, "tf32": 2e-2}     # max abs error of the sigmoid output
RAW_TOL = {"fp32": 2e-4, "tf32": 3e-2}     # relative Frobenius error of pre-BN activations
# Gradients: a forward difference of relative size e flips the LeakyReLU branch of a fraction ~e of the elements, each
# changing its gradient by 80% -> relative Frobenius error ~0.8*sqrt(e) (5e-3 for e = 5e-5 measured in fp32 mode; the
# reference shows the same spread between thread counts, SURVEY.md 7.4).
GRAD_TOL = {"fp32": 3e-2, "tf32": 1e-1}    # relative Frobenius error of weight gradients


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def make_problem(H, W, mode, seed=0, masked=False, skip_channels=4):
    cfg = O.SkipConfig(upsample_mode=mode, skip_channels=skip_channels)
    params = O.init_params(cfg, seed=seed)
    z0 = O.get_noise(32, (H, W), seed=1)
    g = torch.Generator().manual_seed(2)
    target = torch.rand(1, 3, H, W, generator=g)
    mask = (torch.rand(1, 1, H, W, generator=g) > 0.3).float() if masked else None
    return cfg, params, z0, target, mask


def make_engine(cfg, params, H, W, prec):
    import dip_engine as de
    plan = de.Plan(32, 3, cfg.num_scales, 128, cfg.skip_channels, cfg.upsample_mode == "bilinear", H, W,
                   precision=de.PRECISION_TF32 if prec == "tf32" else de.PRECISION_FP32)
    dparams = [p.detach().cuda().contiguous() for p in params]
    dgrads = [torch.zeros_like(p) for p in dparams]
    plan.bind(dparams, dgrads)
    return plan, dparams, dgrads


def is_dead_bias(name):
    # conv bias followed by BatchNorm: gradient is exactly zero in exact arithmetic
    return name.endswith(".b") and "_bn" not in name and not name.startswith("head")


def check_tf32_gradients_like_cudnn(cfg, params, z0, target, dgrads, names):
    """TF32 tier (SURVEY.md 7.4 P1): our error w.r.t. an fp64 oracle must be like the error of the reference's own GPU
    path, i.e. the same graph on torch-CUDA with cuDNN's default TF32 convolutions (comparator only, never shipped).
    At 64x64 the deepest BatchNorms normalise over 4 pixels, so TF32 rounding moves gradients by ~20% for both."""
    p64 = [p.detach().double().requires_grad_(True) for p in params]
    out64 = O.skip_forward(p64, z0.double(), cfg)
    g64 = torch.autograd.grad(O.mse_loss(out64, target.double()), p64)
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        pc = [p.detach().cuda().requires_grad_(True) for p in params]
        gc = torch.autograd.grad(O.mse_loss(O.skip_forward(pc, z0.cuda(), cfg), target.cuda()), pc)
    finally:
        torch.backends.cudnn.allow_tf32 = old
    gmax = max(x.norm().item() for x in g64)
    e_ours, e_cudnn = [], []
    for name, g, c, r in zip(names, dgrads, gc, g64):
        if r.norm().item() < 1e-4 * gmax:
            continue
        eo, ec = rel(g, r), rel(c, r)
        assert eo < 3.0 * ec + 0.08, (name, eo, ec)
        e_ours.append(eo)
        e_cudnn.append(ec)
    assert np.median(e_ours) < 1.5 * np.median(e_cudnn) + 0.01, (np.median(e_ours), np.median(e_cudnn))


@pytest.mark.parametrize("prec", ["fp32", "tf32"])
@pytest.mark.parametrize("shape_mode", [(64, 64, "bilinear", 4), (96, 64, "nearest", 4), (64, 128, "bilinear", 4),
                                        (64, 96, "nearest", 128), (128, 64, "bilinear", 128),
                                        (64, 96, "nearest", 0)])      # num_channels_skip = 0 (no skip branches)
def test_forward_backward_vs_oracle(shape_mode, prec):
    H, W, mode, cs = shape_mode   # cs = 128: the inpainting configuration (BASELINE config 4: skip=128, 256-channel concat)
    cfg, params, z0, target, _ = make_problem(H, W, mode, skip_channels=cs)
    tape = {}
    out_ref = O.skip_forward(params, z0, cfg, tape=tape)
    loss = O.mse_loss(out_ref, target)
    grads_ref = torch.autograd.grad(loss, params)
    dout = (2.0 * (out_ref.detach() - target) / out_ref.numel()).contiguous()

    plan, dparams, dgrads = make_engine(cfg, params, H, W, prec)
    out = plan.forward(z0.cuda())
    torch.cuda.synchronize()
    # pre-BN activations, level by level (localises a broken kernel)
    for l in range(cfg.num_scales):
        for nm in ("raw_s", "raw_d1", "raw_d2", "raw_u", "raw_v")[0 if cs else 1:]:
            ref = tape["L%d.%s" % (l, nm)][0].permute(1, 2, 0)
            got = plan.buffer("L%d.%s" % (l, nm))
            e = rel(got, ref)
            assert e < RAW_TOL[prec], ("L%d.%s" % (l, nm), e)
    err = (out.cpu() - out_ref.detach()).abs().max().item()
    assert err < FWD_TOL[prec], err

    plan.backward(dout.cuda())
    torch.cuda.synchronize()
    names = [n for n, _ in O.param_layout(cfg)]
    gmax = max(gr.norm().item() for gr in grads_ref)
    if prec == "tf32":
        check_tf32_gradients_like_cudnn(cfg, params, z0, target, dgrads, names)
        return
    worst = ("", 0.0)
    for name, g, gr in zip(names, dgrads, grads_ref):
        if gr.norm().item() < 1e-5 * gmax:
            # mathematically-zero gradients (conv bias / concat-BN beta in front of a BatchNorm): rounding noise only
            assert g.norm().item() < 1e-4 * gmax, name
            continue
        e = rel(g, gr)
        if e > worst[1]:
            worst = (name, e)
    assert worst[1] < GRAD_TOL[prec], worst


@pytest.mark.parametrize("prec", ["fp32", "tf32"])
@pytest.mark.parametrize("name", ["denoise64_bilinear_fp32", "inpaint64x96_nearest_masked_skip128_fp32"])
def test_against_reference_golden(name, prec):
    g = np.load(os.path.join(GOLD, name + ".npz"))
    H, W = int(g["H"]), int(g["W"])
    masked = bool(g["masked"])
    cfg, params, z0, target, mask = make_problem(H, W, str(g["mode"]), masked=masked,
                                                 skip_channels=int(g["skip_n11"]) if "skip_n11" in g else 4)
    gn = torch.Generator().manual_seed(123)
    noise = torch.randn(z0.shape, generator=gn)
    plan, dparams, dgrads = make_engine(cfg, params, H, W, prec)
    out = plan.forward(z0.cuda(), noise=noise.cuda(), sigma=float(g["sigma"]))
    torch.cuda.synchronize()
    assert np.abs(out.cpu().numpy() - g["out0"]).max() < FWD_TOL[prec]
    m = mask if masked else torch.ones(1, 1, H, W)
    loss = ((m * (out.cpu() - target)) ** 2).mean().item()
    assert abs(loss - float(g["losses"][0])) < (1e-5 if prec == "fp32" else 1e-3)
    dout = (2.0 * (m * m).cuda() * (out - target.cuda()) / out.numel()).contiguous()
    plan.backward(dout)
    torch.cuda.synchronize()
    if prec == "tf32":
        return  # gradient tier for tf32: test_forward_backward_vs_oracle (cuDNN-TF32 comparator)
    gnorm = np.array([x.double().norm().item() for x in dgrads])
    big = g["gnorm0"] > 1e-5 * g["gnorm0"].max()
    assert np.abs(gnorm[big] / g["gnorm0"][big] - 1).max() < GRAD_TOL[prec]
    assert rel(dgrads[-2].cpu(), torch.from_numpy(g["g_head_w"])) < GRAD_TOL[prec]
    assert rel(dgrads[-10][:4, :8].cpu(), torch.from_numpy(g["g_up0_w_slice"])) < GRAD_TOL[prec]


def test_masked_loss_and_adam_vs_oracle():
    import dip_engine as de
    H, W = 96, 64
    cfg, params, z0, target, mask = make_problem(H, W, "nearest", masked=True)
    plan, dparams, dgrads = make_engine(cfg, params, H, W, "fp32")
    # one oracle step
    out_ref = O.skip_forward(params, z0, cfg)
    loss_ref = O.mse_loss(out_ref, target, mask)
    grads_ref = torch.autograd.grad(loss_ref, params)
    opt = O.Adam(params, 0.01)
    opt.step(grads_ref)
    # engine: forward, fused masked MSE, backward, fused Adam
    out = plan.forward(z0.cuda())
    loss = torch.zeros(1, dtype=torch.float64, device="cuda")
    dout = torch.empty_like(out)
    de.check(de.lib().dip_loss_mse(out.data_ptr(), target.cuda().data_ptr(), mask.cuda().data_ptr(), 3, H * W,
                                   loss.data_ptr(), dout.data_ptr(), None))
    plan.backward(dout)
    for p, gbuf in zip(dparams, dgrads):
        p.grad = gbuf
    adam = de.FusedAdam(dparams, lr=0.01)
    adam.step()
    torch.cuda.synchronize()
    assert abs(loss.item() - loss_ref.item()) < 1e-6
    names = [n for n, _ in O.param_layout(cfg)]
    for name, p, pr in zip(names, dparams, params):
        if is_dead_bias(name) or name.endswith("cat_bn.b") or name.endswith("skip_bn.g"):
            continue  # (near-)zero gradients: the sign of rounding noise decides a full +-lr step (SURVEY.md 7.4)
        d = (p.cpu() - pr.detach()).abs()
        # Adam's first step is +-lr * sign(g): only near-zero gradients may flip
        frac_bad = (d > 1e-3).float().mean().item()
        assert frac_bad < 0.05, (name, frac_bad)


def test_adam_kernel_matches_torch_bitwise_order():
    import dip_engine as de
    g = torch.Generator().manual_seed(0)
    ps = [torch.randn(n, generator=g) for n in (5, 4096, 7001, 128)]
    gs = [[torch.randn(p.shape, generator=g) * 0.1 for p in ps] for _ in range(3)]
    ref = [p.clone().requires_grad_(True) for p in ps]
    topt = torch.optim.Adam(ref, lr=0.01)
    dev = [p.clone().cuda().requires_grad_(True) for p in ps]
    fopt = de.FusedAdam(dev, lr=0.01)
    for step in range(3):
        for r, d, gg in zip(ref, dev, gs[step]):
            r.grad = gg.clone()
            d.grad = gg.cuda()
        topt.step()
        fopt.step()
    torch.cuda.synchronize()
    for r, d in zip(ref, dev):
        assert torch.allclose(r.detach(), d.detach().cpu(), rtol=0, atol=2e-7)


def test_module_api_and_optimize_closure():
    """The notebook-facing path: models.get_net(...).type(dtype), closure, optimize('adam', ...)."""
    import models
    from utils.common_utils import get_noise, get_params, optimize
    dtype = torch.cuda.FloatTensor
    torch.manual_seed(0)
    net = models.get_net(32, "skip", "reflection", skip_n33d=128, skip_n33u=128, skip_n11=4, num_scales=5,
                         upsample_mode="bilinear").type(dtype)
    net.precision = "fp32"
    torch.manual_seed(1)
    z0 = get_noise(32, "noise", (64, 64)).type(dtype).detach()
    gen = torch.Generator().manual_seed(2)
    target = torch.rand(1, 3, 64, 64, generator=gen).type(dtype)
    mse = torch.nn.MSELoss().type(dtype)
    losses = []

    def closure():
        out = net(z0)
        loss = mse(out, target)
        loss.backward()
        losses.append(loss.item())
        return loss

    p = get_params("net", net, z0)
    optimize("adam", p, closure, 0.01, 3)
    # oracle trajectory with the same seeds (no input perturbation)
    cfg, params, z0c, targetc, _ = make_problem(64, 64, "bilinear")
    ref_losses, _ = O.run(cfg, params, z0c, targetc, [None] * 3, 0.0, 0.01)
    assert abs(losses[0] - ref_losses[0]) < 1e-6
    assert abs(losses[1] - ref_losses[1]) < 5e-3   # chaotic from the first Adam step on (SURVEY.md 7.4)
    assert all(np.isfinite(losses))
    # BatchNorm running statistics are maintained like torch does
    sd = net.state_dict()
    assert int(sd["4.num_batches_tracked"]) == 3
    assert float(sd["4.running_var"].mean()) != 1.0


def test_run_iterations_decreases_loss():
    import dip_engine as de
    H, W = 64, 64
    cfg, params, z0, target, _ = make_problem(H, W, "bilinear")
    plan, dparams, dgrads = make_engine(cfg, params, H, W, "tf32")
    for p, gbuf in zip(dparams, dgrads):
        p.grad = gbuf
    adam = de.FusedAdam(dparams, lr=0.01)
    adam._bind(dgrads)
    hist = torch.zeros(40, dtype=torch.float64, device="cuda")
    out = torch.empty(1, 3, H, W, device="cuda")
    de.run_iterations(plan, adam, z0.cuda(), target.cuda(), None, 1. / 30, 7, 40, 0.01, out=out, loss_hist=hist)
    torch.cuda.synchronize()
    h = hist.cpu().numpy()
    assert np.all(np.isfinite(h)) and np.all(h > 0) and h[-5:].mean() < h[:5].mean()
    assert h.max() < 1.0   # one loss per slot (not an accumulated sum)


def test_graph_replayed_forward_backward_equals_eager():
    """dip_forward / dip_backward replay captured CUDA graphs over the plan's staging buffers (notebook path); the
    eager launch sequence (DIP_NO_GRAPH=1) must give the same numbers, and new inputs must be picked up on replay."""
    H, W = 64, 96
    cfg, params, z0, target, _ = make_problem(H, W, "bilinear")
    plan, dparams, dgrads = make_engine(cfg, params, H, W, "tf32")
    zs = [z0.cuda(), (z0 * 0.5 + 0.01).cuda()]
    res = {}
    for mode in ("graph", "graph_again", "eager"):
        if mode == "eager":
            os.environ["DIP_NO_GRAPH"] = "1"
        try:
            for i, z in enumerate(zs):
                out = plan.forward(z)
                dout = (2.0 * (out - target.cuda()) / out.numel()).contiguous()
                plan.backward(dout)
                torch.cuda.synchronize()
                res[(mode, i)] = (out.clone(), [g.clone() for g in dgrads])
        finally:
            os.environ.pop("DIP_NO_GRAPH", None)
    assert not torch.allclose(res[("graph", 0)][0], res[("graph", 1)][0], atol=1e-4)   # the second input was used
    for i in range(2):
        for mode in ("graph_again", "eager"):
            assert torch.allclose(res[("graph", i)][0], res[(mode, i)][0], rtol=0, atol=1e-6)
            for a, b in zip(res[("graph", i)][1], res[(mode, i)][1]):
                assert rel(a, b) < 1e-4 or b.norm().item() < 1e-6


@pytest.mark.parametrize("prec", ["fp32", "tf32"])
def test_inpainting_closure_through_modules_vs_golden(prec):
    """inpainting.ipynb c14-c17 (kate configuration) through the notebook-facing API: skip(32, 3, [128]*5, [128]*5,
    [128]*5, nearest, reflection), total_loss = mse(out * mask, img * mask), optimize('adam', ...)."""
    import models
    from utils.common_utils import get_noise, get_params, optimize
    g = np.load(os.path.join(GOLD, "inpaint64x96_nearest_masked_skip128_fp32.npz"))
    H, W = int(g["H"]), int(g["W"])
    dtype = torch.cuda.FloatTensor
    torch.manual_seed(0)
    net = models.skip(32, 3, num_channels_down=[128] * 5, num_channels_up=[128] * 5, num_channels_skip=[128] * 5,
                      upsample_mode="nearest", need_sigmoid=True, need_bias=True, pad="reflection",
                      act_fun="LeakyReLU").type(dtype)
    net.precision = prec
    torch.manual_seed(1)
    z0 = get_noise(32, "noise", (H, W)).type(dtype).detach()
    gen = torch.Generator().manual_seed(2)
    img_var = torch.rand(1, 3, H, W, generator=gen).type(dtype)
    mask_var = (torch.rand(1, 1, H, W, generator=gen) > 0.3).type(dtype)
    gn = torch.Generator().manual_seed(123)
    mse = torch.nn.MSELoss().type(dtype)
    losses, outs = [], []

    def closure():
        net_input = z0 + torch.randn(z0.shape, generator=gn).type(dtype) * float(g["sigma"])
        out = net(net_input)
        total_loss = mse(out * mask_var, img_var * mask_var)
        total_loss.backward()
        losses.append(total_loss.item())
        outs.append(out.detach())
        return total_loss

    params = get_params("net", net, z0)
    optimize("adam", params, closure, float(g["lr"]), 1)
    gnorm = np.array([p.grad.double().norm().item() for p in params])
    assert np.abs(outs[0].cpu().numpy() - g["out0"]).max() < FWD_TOL[prec]
    assert abs(losses[0] - float(g["losses"][0])) < (1e-5 if prec == "fp32" else 1e-3)
    big = g["gnorm0"] > 1e-4 * g["gnorm0"].max()
    dev = np.abs(gnorm[big] / g["gnorm0"][big] - 1)
    assert (np.median(dev) if prec == "tf32" else dev.max()) < (0.1 if prec == "tf32" else GRAD_TOL[prec]), dev.max()
    optimize("adam", params, closure, float(g["lr"]), 2)           # keeps running (3 iterations like the fixture)
    assert np.isfinite(losses).all() and abs(losses[1] - float(g["losses"][1])) < 2e-2


def test_too_small_an_image_is_refused_like_torch_refuses_it():
    """32 x 64 with 5 scales: the deepest 3x3 conv would reflection-pad a 1 x 2 map; torch raises for the reference's network
    ('Padding size should be less than the corresponding input dimension'), the engine refuses the plan."""
    import dip_engine as de
    with pytest.raises(NotImplementedError, match="at least"):
        de.Plan(32, 3, 5, 128, 4, True, 32, 64)
    de.Plan(32, 3, 5, 128, 4, True, 64, 64)   # the smallest legal size
