"""The device runner (dip_run_iterations: noise -> forward -> MSE -> backward -> Adam, one CUDA graph replayed per
iteration) at a non-zero learning rate, iteration by iteration, against fp64 (H100).

The other runner tests run one iteration at lr = 0 on a fresh plan, where stale weight packs, gradients that accumulate
instead of being overwritten, a wrong Adam step number inside the graph or a wrong loss slot give the right answer.  Here
every configuration makes four calls on one plan and one FusedAdam at lr = 0.01, sigma = 1/30:

    call   iterations   Adam steps taken before
    A      1            0
    B      1            1
    C      3            2
    D      1            5

Before each call the level buffers, every gradient buffer and the weight-gradient partials ("wacc", tensor-core modes)
are filled with NaN, and p, m, v are copied.  After each call:

* stages: every stage and every parameter gradient through TS.check (the stage references of tests/stage_ref.py at the
  configuration's padding and activation; the tolerances of tests/test_stages_gpu.py) at the parameters the last
  iteration's forward used: the copy taken before a one-iteration call, and for C the parameters reconstructed from the state the call left (below).  Stale weight packs fail the convolutions by orders of
  magnitude; a gradient that accumulates or is not written fails its 'grad:' entry or comes out NaN;
* Adam (one-iteration calls): from the copied p, m, v, the gradients the call left and step = steps before + 1,
      m* = b1 m + (1 - b1) g,  v* = b2 v + (1 - b2) g^2          (fp64)
  and the engine's m', v' must be within 4u (|b1 m| + |(1 - b1) g|) and 4u (b2 v + (1 - b2) g^2) of them (u = 2^-24; one
  rounding each for the fp32 constant 1 - b1 (or b2), the product, the second product and the sum; + 2^-149 where
  v* < 2^-126).  Then U = (lr / bc1) m' / (sqrt(v') / sqrt(bc2) + eps), bc = 1 - b^step, in fp64 from the engine's own m'
  and v', and p' must be within u |p - U| + 8u |U| of p - U (k_adam rounds lr / bc1, sqrt(bc2), sqrt(v'), the division,
  the eps sum, m' / denom and the product once each: 7u, and the final subtraction u |p - U|).  Where m' == 0, p' == p
  exactly;
* C, the last of three iterations: the parameters its forward used are p_C + U(m_C, v_C, step 5), reconstructed in fp64
  from the engine's state after the call.  With U_k the kernel's own update, p_C = fl(x - U_k) and |U_k - U| <= 7u |U|,
  so the reconstruction is within delta = 2u |p_C| + 8u |U| of the true x.  stage_ref adds that uncertainty to the
  tolerance of every convolution that multiplies a parameter: conv(|input|, delta_w) + delta_b (conv_transpose for the
  input gradients); in bf16 mode the tensor-core convolutions multiply bf16(x), so their weight uncertainty is
  bf16(x + delta) - bf16(x - delta), one bf16 ulp where a rounding boundary lies within delta of x, 0 elsewhere.  A wrong
  step number, or packs of the weights of an earlier iteration, reconstructs parameters that are off by a whole Adam
  step and the convolutions fail;
* loss slots: every slot written is finite and > 0, the ones after it keep the -1 they were filled with, and the last
  iteration's slot is the fp64 MSE of the engine's output (through O.downsample for super-resolution, with the mask for
  inpainting).  Bound: k_mse sums d^2, d = m (out - target) in fp32 (d^2 carries 2 roundings), k = ceil(n / (256 blocks))
  fma terms per thread, a 5-level warp tree and a 5-level block tree, then multiplies by fl(1 / n) (1 rounding): every
  term passes through at most k + 13 roundings of a sum of non-negative terms, so the fp32 block sums are within
  gamma_{k+13} = (k + 13) u / (1 - (k + 13) u) of the exact sum relative to it.  Each block's term is then rounded to a
  multiple of 2^-48 (at most 2^-49 each; the fp64 atomics on multiples of 2^-48 below 32 are exact): tolerance
  gamma_{k+13} (L + D) + D + blocks 2^-49.  D = 0 except for super-resolution, where the fp32 downsampled output y is
  within e = gamma_{K^2+1} (|kernel| * |out|) of the fp64 one (K^2 fma terms and the fp32 taps), and the MSE moves by
  at most D = mean(2 |y - t| e + e^2);
* noise: the padded level-0 input is pad(dip_noise_perturb(offset = steps before + iterations - 1)) bit for bit, with
  exact zeros in the stored depth's extra channels.

The same four calls run through the eager loop (DIP_NO_GRAPH=1), two through the timed eager pass without side streams
(what bench.py's roofline pass runs), and the notebook path (models + utils.optimize, graph-replayed dip_forward /
dip_backward) is checked stage by stage after a FusedAdam step.  The Adam kernel on its own is checked against the same
fp64 bounds on the flagship layout plus tensors at its 2048-element chunk edges, at gradient scales 1e-6 .. 1e2, with
exact-zero gradients, at steps 1, 2, 3, 2000 and 100000, for torch's defaults and for other hyper-parameters.
"""
import contextlib
import math
import os

import pytest
import torch

from oracle import dip_oracle as O
import envelope_cases as E
import stage_ref as SR
import test_stages_gpu as TS

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
LR, SIGMA, SEED = 0.01, TS.SIGMA, TS.SEED
BETAS, EPS = (0.9, 0.999), 1e-8
CALLS = [("A", 1, 0), ("B", 1, 1), ("C", 3, 2), ("D", 1, 5)]   # (call, iterations, Adam steps taken before)
HIST = 5                       # loss_hist slots; every call leaves the ones after its iterations at -1
MSE_BLOCK_CAP = 4 * 132        # launch_mse (kernels_mem.cu): min(ceil(n / 256), 4 kNumSms) blocks of 256 threads
ADAM = {}                      # tag -> {'m' | 'v' | 'p': worst |err| / bound}
LOSS = {}                      # mode -> worst |slot - fp64 MSE| / bound

# (id, task, SkipConfig, H, W, precision mode): the comment names what only that configuration reaches
CONFIGS = [
    # the flagship schedule: deferred weight gradients and side streams
    ("denoise_cs4_tf32", "denoise", lambda: E.cfg_of("cs4"), 128, 128, "tf32"),
    # bf16 weight twins repacked every iteration
    ("denoise_cs4_bf16", "denoise", lambda: E.cfg_of("cs4"), 128, 128, "bf16"),
    # the SIMT convolutions, each weight gradient summed by k_wgrad_unpack_table on its own entry
    ("denoise_cs4_fp32", "denoise", lambda: E.cfg_of("cs4"), 64, 96, "fp32"),
    # the two-part up-conv weight gradient (up_a / up_b) into one tensor; the masked loss
    ("inpaint_cs128_tf32", "inpaint", lambda: E.cfg_of("cs128"), 128, 192, "tf32"),
    # ds_y / ds_dy and the loss on the low-resolution output
    ("sr_cs4_bf16", "sr", lambda: E.cfg_of("cs4"), 256, 256, "bf16"),
    # skinny 1x1 convolutions with fp64-atomic weight gradients
    ("denoise_snail_tf32", "denoise", lambda: E.cfg_of("snail"), 64, 96, "tf32"),
    # W % 4 = 2: the separate k_noise -> zbuf path
    ("denoise_L1_tf32", "denoise", lambda: E.cfg_of("L1"), 10, 14, "tf32"),
    # zero padding (k_noise_pad<true>) and the templated BatchNorm kernels of Swish over several iterations
    ("denoise_skipdefault_swish_tf32", "denoise", lambda: E.cfg_of("skipdefault", "zero", "Swish"), 64, 96, "tf32"),
]
BY_ID = {c[0]: c[1:] for c in CONFIGS}


@contextlib.contextmanager
def environment(**values):
    saved = {k: os.environ.get(k) for k in values}
    os.environ.update(values)
    try:
        yield
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def gamma(n):
    return n * U / (1 - n * U)


def flat(ts):
    return torch.cat([t.reshape(-1) for t in ts])


def unflat(x, like):
    out, o = [], 0
    for t in like:
        out.append(x[o:o + t.numel()].view(t.shape))
        o += t.numel()
    return out


def poison(plan, L, grads, mode):
    """NaN into every level buffer, the weight-gradient partials and the gradient buffers: whatever a call reads without
    writing it first shows up as NaN"""
    TS.fill_nan(plan, L)
    wacc = TS.buffer_view(plan, "wacc")
    assert (wacc is None) == (mode == "fp32"), "the tensor-core modes register their weight-gradient partials as 'wacc'"
    if wacc is not None:
        wacc.fill_(float("nan"))
    for g in grads:
        g.fill_(float("nan"))
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ Adam
def adam_update(m, v, lr, betas, eps, step):
    """U of p' = p - U in fp64 (torch.optim.Adam's step from the updated m, v)"""
    bc1, bc2 = 1 - betas[0] ** step, 1 - betas[1] ** step
    return (lr / bc1) * m / (v.sqrt() / math.sqrt(bc2) + eps)


def check_adam(tag, before, g, after, lr, betas, eps, step):
    """before / after: flat (p, m, v) around one Adam step with gradient g (module docstring)"""
    b1, b2 = betas
    p0, m0, v0 = (t.double() for t in before)
    p1, m1, v1 = (t.double() for t in after)
    g = g.double()
    ms = b1 * m0 + (1 - b1) * g
    tm = 4 * U * ((b1 * m0).abs() + ((1 - b1) * g).abs())
    vs = b2 * v0 + (1 - b2) * g * g
    tv = 4 * U * vs + (vs < 2.0 ** -126).double() * 2.0 ** -149
    upd = adam_update(m1, v1, lr, betas, eps, step)
    ps = p0 - upd
    tp = U * ps.abs() + 8 * U * upd.abs()
    row = ADAM.setdefault(tag, {})
    failures = []
    for q, got, ref, tol in (("m", m1, ms, tm), ("v", v1, vs, tv), ("p", p1, ps, tp)):
        if not torch.isfinite(got).all():
            failures.append("%s: %d non-finite elements" % (q, (~torch.isfinite(got)).sum().item()))
            continue
        d = (got - ref).abs()
        r = torch.where(d == 0, torch.zeros_like(d), d / tol)
        worst = r.max().item()
        row[q] = max(row.get(q, 0.0), worst)
        if not worst <= 1.0:
            i = r.argmax().item()
            failures.append("%s: worst |err|/bound = %.3g at flat element %d (got %.9g, fp64 %.9g, bound %.3g; g %.3g)" % (
                q, worst, i, got[i].item(), ref[i].item(), tol[i].item(), g[i].item()))
    still = m1 == 0
    if not torch.equal(p1[still], p0[still]):
        failures.append("p changed at %d elements where m' == 0" % (p1[still] != p0[still]).sum().item())
    assert not failures, "[Adam %s, step %d]\n  " % (tag, step) + "\n  ".join(failures)


# ------------------------------------------------------------------------------------------------ the runner
class Runner(TS.Runner):
    """the plan, FusedAdam and inputs of a runner configuration (test_stages_gpu.Runner) at lr = LR"""

    def __init__(self, cid):
        task, make_cfg, H, W, mode = BY_ID[cid]
        super().__init__(make_cfg(), H, W, mode, task, LR)
        self.cid = cid
        self.hist = torch.empty(HIST, dtype=torch.float64, device="cuda")

    def call(self, name, iters, step0):
        """one dip_run_iterations call from poisoned buffers, then every check of the module docstring"""
        import dip_engine as de
        cfg, adam = self.cfg, self.adam
        tag = "%s call %s (%d iteration%s after %d steps)" % (self.cid, name, iters, "s" if iters > 1 else "", step0)
        assert adam.step_count == step0
        poison(self.plan, cfg.num_scales, self.grads, self.mode)
        before = (flat(self.params).clone(), adam.m_flat.clone(), adam.v_flat.clone())
        self.hist.fill_(-1.0)
        de.run_iterations(self.plan, adam, self.z0, self.target, self.mask, SIGMA, SEED, iters, LR, out=self.out,
                          loss_hist=self.hist)
        torch.cuda.synchronize()
        assert adam.step_count == step0 + iters
        self.check_pin(tag, step0 + iters - 1)
        self.check_slots(tag, iters)
        if iters == 1:
            self.check_stages(tag, unflat(before[0], self.params))
            check_adam("runner", before, flat(self.grads), (flat(self.params), adam.m_flat, adam.v_flat), LR, BETAS, EPS,
                       step0 + 1)
        else:   # the parameters of the last iteration's forward, from the state the call left
            p, m, v = flat(self.params).double(), adam.m_flat.double(), adam.v_flat.double()
            upd = adam_update(m, v, LR, BETAS, EPS, step0 + iters)
            delta = 2 * U * p.abs() + 8 * U * upd.abs()
            self.check_stages(tag, unflat(p + upd, self.params), unflat(delta, self.params))

    def check_slots(self, tag, iters):
        h = self.hist.cpu()
        assert torch.isfinite(h[:iters]).all() and (h[:iters] > 0).all(), "[%s] loss slots %s" % (tag, h.tolist())
        assert (h[iters:] == -1).all(), "[%s] slots after the call's iterations were written: %s" % (tag, h.tolist())
        o, t = self.out.double().cpu(), self.target.double().cpu()
        mask = None if self.mask is None else self.mask.double().cpu()
        if self.down is None:
            y, e = o, torch.zeros_like(o)
        else:
            kern, f, pad = self.down
            y = O.downsample(o, kern, f, pad)
            e = gamma(kern.numel() + 1) * O.downsample(o.abs(), kern.abs(), f, pad)
        ref = O.mse_loss(y, t, mask).item()
        n = y.numel()
        mm = 1.0 if mask is None else mask
        d, em = (mm * (y - t)).abs(), mm * e
        D = ((2 * d * em + em * em).sum() / n).item()
        blocks = min(-(-n // 256), MSE_BLOCK_CAP)
        k = -(-n // (256 * blocks))
        tol = gamma(k + 13) * (ref + D) + D + blocks * 2.0 ** -49
        got = h[iters - 1].item()
        LOSS[self.mode] = max(LOSS.get(self.mode, 0.0), abs(got - ref) / tol)
        assert abs(got - ref) <= tol, "[%s] loss slot %d = %.17g, fp64 MSE of the output %.17g, bound %.3g" % (
            tag, iters - 1, got, ref, tol)


def print_tables():
    TS.print_table()
    for tag, row in sorted(ADAM.items()):
        print("[runner steps] Adam %s, worst |err|/bound: m %.3g, v %.3g, p %.3g" % (tag, row["m"], row["v"], row["p"]))
    if LOSS:
        print("[runner steps] loss slot, worst |err|/bound: %s" % ", ".join("%s %.3g" % kv for kv in sorted(LOSS.items())))


@pytest.mark.parametrize("cid", [c[0] for c in CONFIGS])
def test_runner_calls_step_by_step(cid):
    r = Runner(cid)
    if r.mode == "fp32":
        with pytest.raises(RuntimeError, match="unknown buffer wacc"):
            r.plan.buffer("wacc")
    for name, iters, step0 in CALLS:
        r.call(name, iters, step0)
    assert r.adam.step_count == 6
    print_tables()


def test_runner_calls_eager_loop():
    """the eager loop (DIP_NO_GRAPH=1): step, noise stream and loss slot come from the host"""
    with environment(DIP_NO_GRAPH="1"):
        r = Runner("denoise_cs4_tf32")
        for name, iters, step0 in CALLS:
            r.call(name, iters, step0)
    assert r.adam.step_count == 6
    print_tables()


def test_runner_calls_timed_without_side_streams():
    """what bench.py's roofline pass runs: timing events around every launch (eager), no side streams"""
    with environment(DIP_NO_SIDE="1"):
        r = Runner("denoise_cs4_tf32")
        r.plan.set_timing(True)
        try:
            for name, iters, step0 in CALLS[:2]:
                r.call(name, iters, step0)
            assert len(r.plan.get_timing_records()) > 0
        finally:
            r.plan.set_timing(False)
    assert r.adam.step_count == 2
    print_tables()


def test_module_path_after_an_adam_step():
    """models + utils.optimize('adam'): the second closure's graph-replayed dip_forward / dip_backward, from NaN-filled
    buffers and gradients, checked stage by stage at the parameters it ran with (those after the first FusedAdam step)"""
    import models
    from utils.common_utils import optimize
    cfg = E.cfg_of("cs4")
    H, W = 128, 128
    torch.manual_seed(0)
    net = models.get_net(32, "skip", "reflection", skip_n33d=128, skip_n33u=128, skip_n11=4, num_scales=5,
                         upsample_mode="bilinear").type(torch.cuda.FloatTensor)
    assert net.precision == "tf32"
    params = list(net.parameters())
    with torch.no_grad():
        for p, v in zip(params, TS.params_for(cfg, 3)):
            assert p.shape == v.shape
            p.copy_(v)
    g = torch.Generator().manual_seed(5)
    # (U(0, 1), as every stage test: at get_noise's U(0, 0.1) the level-0 d1 BatchNorm reached 1.7x the forward bound
    # of stage_ref, whose BatchNorm tolerance does not model the error of the statistics when |mean| >> std)
    z0 = torch.rand(1, 32, H, W, generator=g).cuda()
    target = torch.rand(1, 3, H, W, generator=g).cuda()
    mse = torch.nn.MSELoss()
    seen = {"calls": 0}

    def closure():
        seen["calls"] += 1
        second = seen["calls"] == 2
        if second:
            seen["params"] = [p.detach().clone() for p in params]
            poison(list(net._dip_plans.values())[0], cfg.num_scales, [net._dip_grad_arena], "tf32")
        out = net(z0)
        if second:
            seen["out"] = out
            out.register_hook(lambda d: seen.__setitem__("dout", d.detach().clone()))
        loss = mse(out, target)
        loss.backward()
        return loss

    optimize("adam", params, closure, LR, 2)
    torch.cuda.synchronize()
    assert seen["calls"] == 2 and len(net._dip_plans) == 1
    assert not all(torch.equal(a, b) for a, b in zip(seen["params"], params)), "the first Adam step moved nothing"
    plan = list(net._dip_plans.values())[0]
    out = seen["out"].detach()
    refs = SR.Refs()
    rd = TS.engine_src(plan, "tf32", out)
    SR.forward(cfg, seen["params"], rd, "tf32", refs, z=z0)
    SR.backward(cfg, seen["params"], rd, "tf32", refs, seen["dout"][0])
    TS.check("module path, second closure", cfg, "tf32", plan, refs, [p.grad for p in params], out)
    print_tables()


# ------------------------------------------------------------------------------------------------ the Adam kernel
ADAM_SETTINGS = [dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8), dict(lr=3e-3, betas=(0.8, 0.99), eps=1e-6)]


@pytest.mark.parametrize("hyper", ADAM_SETTINGS, ids=["defaults", "lr3e-3_betas0.8_0.99_eps1e-6"])
def test_adam_kernel_at_its_edges(hyper):
    """FusedAdam.step (dip_adam_step) on the flagship network's parameter layout plus tensors around the 2048-element
    chunks of k_adam; per-tensor gradient scales 1e-6 .. 1e2, one tensor of exact zeros (a dead bias), one with every
    other element exactly zero; steps 1, 2, 3, then 2000 and 100000; every step against the fp64 bounds above"""
    import dip_engine as de
    cfg = E.cfg_of("cs4")
    names = [n for n, _ in O.param_layout(cfg)] + ["extra%d" % k for k in (1, 3, 2047, 2048, 2049, 4097, 147461)]
    numels = [math.prod(s) for _, s in O.param_layout(cfg)] + [1, 3, 2047, 2048, 2049, 4097, 147461]
    zero, half = names.index("L0.d1.b"), names.index("L0.d2.w")
    gen = torch.Generator().manual_seed(11)
    params = [(0.1 * torch.randn(k, generator=gen)).cuda() for k in numels]
    grads = [torch.empty_like(p) for p in params]
    for p, gb in zip(params, grads):
        p.grad = gb
    scales = torch.logspace(-6, 2, len(numels), dtype=torch.float64)[torch.randperm(len(numels), generator=gen)]
    adam = de.FusedAdam(params, **hyper)
    tag = "kernel lr %g betas %s eps %g" % (hyper["lr"], hyper["betas"], hyper["eps"])
    for taken in (0, 1, 2, 1999, 99999):
        adam.step_count = taken
        for i, gb in enumerate(grads):
            gb.copy_((torch.randn(numels[i], generator=gen, dtype=torch.float64) * scales[i]).float())
        grads[zero].zero_()
        grads[half][::2] = 0.0
        before = (flat(params).clone(), adam.m_flat.clone(), adam.v_flat.clone())
        adam.step()
        torch.cuda.synchronize()
        check_adam(tag, before, flat(grads), (flat(params), adam.m_flat, adam.v_flat), hyper["lr"], hyper["betas"],
                   hyper["eps"], taken + 1)
        assert not adam.m[zero].any() and torch.equal(params[zero], unflat(before[0], params)[zero])
    print_tables()


def test_runner_refuses_betas_and_eps_it_does_not_use():
    """dip_run_iterations steps Adam with torch's defaults: an optimiser with other betas or eps is refused before
    anything is launched, and one with the defaults runs"""
    import dip_engine as de
    r = Runner("denoise_L1_tf32")
    p0 = [p.clone() for p in r.params]
    for kw, field in ((dict(betas=(0.8, 0.99)), "betas"), (dict(betas=(0.9, 0.99)), "betas"), (dict(eps=1e-6), "eps")):
        adam = de.FusedAdam(r.params, lr=LR, **kw)
        adam._bind(r.grads)
        with pytest.raises(ValueError, match=field):
            de.run_iterations(r.plan, adam, r.z0, r.target, None, SIGMA, SEED, 1, LR, out=r.out)
        assert adam.step_count == 0
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(p0, r.params))
        assert not adam.m_flat.any() and not adam.v_flat.any()
    de.run_iterations(r.plan, r.adam, r.z0, r.target, None, SIGMA, SEED, 1, LR, out=r.out)
    torch.cuda.synchronize()
    assert r.adam.step_count == 1
    assert not all(torch.equal(a, b) for a, b in zip(p0, r.params))
    assert all(torch.isfinite(p).all() for p in r.params)
