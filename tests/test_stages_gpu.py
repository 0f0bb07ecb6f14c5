"""P1 stage tier: one forward + backward on the GPU, then every stage of the step checked on its own (teacher forcing).

Each stage's reference (tests/stage_ref.py) is computed in fp64 on the GPU from the engine's own input buffers of that
stage, so no error carries over from earlier stages and no LeakyReLU branch flips: the tolerance is the rounding of that
one stage, element by element (convolutions: 2 (e_op + n 2^-23) M; memory-bound stages: 1e-5 |ref| + 3e-5 s_c; see the
module docstring of stage_ref.py).  Parameters are away from init (random gamma, beta and biases, different for the
skip and up channels of every concat BN), and every registered buffer is filled with NaN before the first pass, so a
halo cell, tail or tile edge that no kernel writes shows up as a non-finite stage output.  Every network runs with
its own padding and activation (SkipConfig.pad / act_fun): with zero padding the halo ring of every padded conv input and
of its bf16 twin must hold exact zeros, and an activation other than LeakyReLU (no jump in its derivative) may not
exclude a single element from the backward checks.

The same machinery judges the zero-padded networks (tests/test_zero_pad_gpu.py), the other activations
(tests/test_act_fun_gpu.py), the envelope table (tests/test_envelope_gpu.py) and the device runner at a non-zero learning
rate (tests/test_runner_steps_gpu.py).
"""
import ctypes

import pytest
import torch

from oracle import dip_oracle as O
import envelope_cases as E
import stage_ref as SR

pytestmark = pytest.mark.gpu
MODES = ["fp32", "tf32", "bf16"]
SIGMA, SEED = 1. / 30, 7   # the runner's noise: z0 + sigma * N(0, 1) from stream (SEED, iteration offset)
LEVEL_BUFFERS = ["Pin", "raw_s", "raw_d1", "rawF", "P_d1", "raw_d2", "P_d2", "P_cat", "raw_u", "A_u", "raw_v", "U",
                 "dRaw_v", "dA_u", "dRaw_u", "dP_cat", "dCat", "dRaw_s", "dUp", "dS", "dRaw_d2", "dP_d1", "dRaw_d1",
                 "dRawF", "dPin", "Pin16", "P_d1_16", "P_d2_16", "P_cat16", "A_u16", "dRaw_v16", "dRaw_u16", "dRaw_d2_16",
                 "dRaw_d1_16", "dRaw_s16", "dRawF16"]
WORST = {}   # mode -> {stage: worst |err| / tolerance}
FROB = {}    # mode -> {conv stage: worst relative Frobenius error / its bound}


def make_plan(cfg, H, W, mode, input_grad=False):
    """dip_engine.Plan of an oracle SkipConfig: per-scale down / up / skip widths and up modes, downsampling, padding and
    activation"""
    import dip_engine as de
    prec = {"fp32": de.PRECISION_FP32, "tf32": de.PRECISION_TF32, "bf16": de.PRECISION_BF16}[mode]
    L = cfg.num_scales
    return de.Plan(cfg.in_channels, cfg.out_channels, L, [cfg.nd(l) for l in range(L)], [cfg.ns(l) for l in range(L)],
                   [SR._up_mode(cfg, l) for l in range(L)], H, W, precision=prec, need_sigmoid=cfg.need_sigmoid,
                   input_grad=input_grad, channels_up=[cfg.nu(l) for l in range(L)], downsample_mode=cfg.downsample_mode,
                   pad=cfg.pad, act=cfg.act_fun)


def engine_src(plan, mode, out):
    """src(name) of stage_ref over the engine's buffers (bf16 twins as registered views) and its output"""
    src = plan.buffer if mode != "bf16" else (lambda n: buffer_view(plan, n) if n.endswith("16") else plan.buffer(n))
    return lambda n: out[0] if n == "out" else src(n)


def buffer_view(plan, name):
    """the registered buffer's [:, :, :c] region inside the workspace (a view; Plan.buffer returns a copy), or None"""
    import dip_engine as de
    p = ctypes.c_void_p()
    dims = (ctypes.c_int * 4)()
    if de.lib().dip_plan_buffer(plan.h, name.encode(), ctypes.byref(p), dims) != 0:
        return None
    rows, cols, ld, c = dims[0], dims[1], dims[2], dims[3]
    esz = 2 if name.endswith("16") else 4
    off = p.value - plan.workspace.data_ptr()
    flat = plan.workspace[off:off + rows * cols * ld * esz].view(torch.bfloat16 if esz == 2 else torch.float32)
    return flat.view(rows, cols, ld)[:, :, :c]


def fill_nan(plan, L):
    n = 0
    for l in range(L):
        for b in LEVEL_BUFFERS:
            v = buffer_view(plan, "L%d.%s" % (l, b))
            if v is not None and v.numel():
                v.fill_(float("nan"))
                n += 1
    torch.cuda.synchronize()
    assert n > 0


def fp32_dropped(cfg, name):
    """bf16 mode keeps only the bf16 twin of these stage outputs (DESIGN.md section 2; engine.cu fwd_level / bn_bwd)"""
    l, b = int(name[1]), name.split(".", 1)[1]
    if b in ("P_d1", "A_u", "dRaw_v", "dRaw_u", "dRaw_d2", "dRawF"):
        return True
    if b == "dRaw_d1":
        return cfg.downsample_mode != "avg"
    if b == "dRaw_s":
        return cfg.ns(l) == 128
    if b == "P_d2":
        return l < cfg.num_scales - 1 and cfg.ns(l + 1) != 4
    return False


def bf16_ulp(x):
    a = x.abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


def ratio_of(got, ref, tol, excl):
    d = (got.double() - ref).abs()
    r = torch.where(d == 0, torch.zeros_like(d), d / tol.expand_as(d))
    if excl is not None:
        r = torch.where(excl, torch.zeros_like(r), r)
    return r


HALO_BUFFERS = ["Pin", "P_d1", "P_d2", "P_cat", "Pin16", "P_d1_16", "P_d2_16", "P_cat16"]


def check_halos(cfg, mode, plan):
    """the halo ring of every padded conv input (and of its bf16 twin) holds exact zeros"""
    bad, n = [], 0
    for l in range(cfg.num_scales):
        for b in HALO_BUFFERS:
            name = "L%d.%s" % (l, b)
            if b.startswith("P_d2") and l == cfg.num_scales - 1:
                continue   # the deepest level's P_d2 is plain (no conv reads it padded)
            if mode == "bf16" and not b.endswith("16") and (
                    fp32_dropped(cfg, name) or (b == "Pin" and l > 0 and fp32_dropped(cfg, "L%d.P_d2" % (l - 1)))):
                continue   # never written in bf16 mode (its twin is checked; a level's Pin is the P_d2 of the level above)
            v = buffer_view(plan, name)
            if v is None or not v.numel():
                continue
            v = v.float()
            ring = torch.cat([v[0].flatten(), v[-1].flatten(), v[:, 0].flatten(), v[:, -1].flatten()])
            n += 1
            if not torch.equal(ring, torch.zeros_like(ring)):
                bad.append("%s: %d non-zero halo cells" % (name, (ring != 0).sum().item()))
    assert n > 0
    assert not bad, "[%s] " % mode + "; ".join(bad)


def check_no_exclusion(refs):
    """no activation but LeakyReLU has a jump in its derivative: not one element may be excluded from the backward checks"""
    assert refs.excl, "no BN(+act) backward was checked"
    shares = {name: frac for name, (frac, _) in refs.excl.items()}
    assert all(frac == 0.0 for frac in shares.values()), shares
    assert all(e is None or not e.any() for _, _, e in refs.d.values())


def check(tag, cfg, mode, plan, refs, dgrads, out, dz=None):
    """every stage of `refs` against the engine's buffers, gradients, output and dz (module docstring)"""
    if cfg.pad != "reflection":
        check_halos(cfg, mode, plan)
    if cfg.act_fun != "LeakyReLU":
        check_no_exclusion(refs)
    names = [n for n, _ in O.param_layout(cfg)]
    table = WORST.setdefault(mode, {})
    failures = []
    for name, (ref, tol, excl) in refs.d.items():
        if name.startswith("grad:"):
            got = dgrads[names.index(name[5:])].double()
        elif name == "out":
            got = out[0].double()
        elif name == "dz":
            got = dz.double()
        elif mode == "bf16" and fp32_dropped(cfg, name):
            got = None
        else:
            got = plan.buffer(name).double()
        if mode == "bf16" and not name.startswith("grad:") and name not in ("out", "dz"):
            twin = buffer_view(plan, SR._twin(name))
            if twin is not None:
                twin = twin.double()
                if got is not None:   # the twin of a kept fp32 tensor is its round-to-nearest-even copy
                    if not torch.equal(twin, SR.bf16(got)):
                        failures.append("%s: bf16 twin != bf16(fp32 tensor)" % name)
                else:                 # only the twin exists: one bf16 ulp of the rounded reference, few elements differ
                    rb = SR.bf16(ref)
                    d = (twin - rb).abs()
                    bad = d > bf16_ulp(rb) + 2 * tol
                    if excl is not None:
                        bad &= ~excl
                    if not torch.isfinite(twin).all() or bad.any() or (d > 0).sum().item() > 1e-2 * d.numel() + 8:
                        failures.append("%s (bf16 twin): %d elements beyond one ulp, %d differ of %d" % (
                            name, bad.sum().item(), (d > 0).sum().item(), d.numel()))
                    continue
        if got is None:   # a stage that bf16 mode keeps as a twin only, but whose twin is not registered: unchecked
            failures.append("%s: fp32 tensor dropped in bf16 mode, but no bf16 twin %s is registered" % (name, SR._twin(name)))
            continue
        if not torch.isfinite(got).all():
            idx = (~torch.isfinite(got)).nonzero()[0].tolist()
            failures.append("%s: %d non-finite elements (unwritten memory?), first at %s" % (
                name, (~torch.isfinite(got)).sum().item(), idx))
            continue
        r = ratio_of(got, ref, tol, excl)
        worst = r.max().item()
        key = name.split(".", 1)[1] if name.startswith("L") else name
        key = "grad:" + name.split(".", 1)[1] if name.startswith("grad:L") else key
        table[key] = max(table.get(key, 0.0), worst)
        if name in refs.conv:   # convolutions: relative Frobenius error at the precision the kernel runs in
            bound = SR.FROB_TOL[refs.conv[name]]
            dn, rn = (got - ref).norm().item(), ref.norm().item()
            fro = dn / rn if rn > 0 else (0.0 if dn == 0 else float("inf"))
            ftab = FROB.setdefault(mode, {})
            ftab[key] = max(ftab.get(key, (0.0, 0.0)), (fro / bound, fro))
            if not fro <= bound:
                failures.append("%s: relative Frobenius error %.3g > %.1g (%s kernel)" % (name, fro, bound, refs.conv[name]))
        if not worst <= 1.0:
            i = tuple(torch.unravel_index(r.argmax(), r.shape))
            i = tuple(int(x) for x in i)
            failures.append("%s: worst |err|/tol = %.3g at %s (got %.9g ref %.9g tol %.3g)" % (
                name, worst, i, got[i].item(), ref[i].item(), tol.expand_as(r)[i].item()))
    for name, (frac, n) in refs.excl.items():   # (one element may sit there in the 768 of a 2 x 3 x 128 map)
        if frac >= 1e-3 + 1.5 / n:
            failures.append("%s: %.2g of the elements sit at the LeakyReLU boundary" % (name, frac))
    assert not failures, "[%s %s]\n  " % (tag, mode) + "\n  ".join(failures)


def params_for(cfg, seed=0):
    return [p.float() for p in SR.random_affine(cfg, O.init_params(cfg, seed=seed), seed=seed + 11)]


def run_direct(cfg, H, W, mode, input_grad=False, seed=0):
    """plan.forward / plan.backward with dout = the MSE gradient against a random target; every stage checked"""
    params = params_for(cfg, seed)
    g = torch.Generator().manual_seed(seed + 1)
    z = torch.rand(1, cfg.in_channels, H, W, generator=g).cuda()
    target = torch.rand(1, cfg.out_channels, H, W, generator=g).cuda()
    plan = make_plan(cfg, H, W, mode, input_grad)
    dparams = [p.cuda().contiguous() for p in params]
    dgrads = [torch.zeros_like(p) for p in dparams]
    plan.bind(dparams, dgrads)
    fill_nan(plan, cfg.num_scales)
    out = plan.forward(z)
    dout = (2.0 * (out - target) / out.numel()).contiguous()
    plan.backward(dout)
    dz = plan.input_grad() if input_grad else None
    torch.cuda.synchronize()
    refs = SR.Refs()
    rd = engine_src(plan, mode, out)
    SR.forward(cfg, dparams, rd, mode, refs, z=z)
    SR.backward(cfg, dparams, rd, mode, refs, dout[0], input_grad=input_grad)
    check("%s %dx%d" % (cfg_tag(cfg), H, W), cfg, mode, plan, refs, dgrads, out, dz)


def cfg_tag(cfg):
    return "in%d out%d ch%s up%s skip%s %s %s pad=%s %s" % (
        cfg.in_channels, cfg.out_channels, cfg.channels, cfg.channels_up, cfg.skip_channels, cfg.upsample_mode,
        cfg.downsample_mode, cfg.pad, cfg.act_fun)


def print_table():
    for mode in MODES:
        if mode in WORST:
            row = sorted(WORST[mode].items())
            print("\n[stage tier %s] worst |err|/tol per stage: %s" % (mode, ", ".join("%s %.2g" % kv for kv in row)))
        if mode in FROB:
            row = sorted(FROB[mode].items())
            print("[stage tier %s] conv stages, worst relative Frobenius error (/ its bound): %s" % (
                mode, ", ".join("%s %.2g (%.2g)" % (k, v[1], v[0]) for k, v in row)))


CASES = [("cs4", 64, 96, False), ("cs128", 96, 64, False), ("cs0", 64, 96, False), ("snail", 64, 96, False),
         ("kate", 96, 64, False), ("modes", 64, 96, False), ("ingrad", 64, 96, True), ("cs4", 256, 384, False),
         ("avg128", 64, 96, False), ("per_scale128", 64, 96, False)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", CASES, ids=["%s_%dx%d" % c[:3] for c in CASES])
def test_every_stage_direct(case, mode):
    kind, H, W, input_grad = case
    run_direct(E.cfg_of(kind), H, W, mode, input_grad)
    print_table()


def test_every_stage_flagship_512_tf32():
    run_direct(E.cfg_of("cs4"), 512, 512, "tf32")
    print_table()


class Runner:
    """one plan, one FusedAdam at lr and the inputs of a device-runner configuration: z0 and the target U(0, 1) (the
    target at the x4 Lanczos2-downsampled size for task 'sr'), a random mask for 'inpaint', the parameters of
    params_for(cfg, 3) bound as the gradient buffers' owners"""

    def __init__(self, cfg, H, W, mode, task, lr):
        import dip_engine as de
        self.cfg, self.mode, self.task = cfg, mode, task
        g = torch.Generator().manual_seed(5)
        self.z0 = torch.rand(1, cfg.in_channels, H, W, generator=g).cuda()
        self.plan = make_plan(cfg, H, W, mode)
        self.mask = self.down = None
        if task == "sr":
            kern = O.down_kernel(4, "lanczos2", 0.5)
            self.down = (torch.from_numpy(kern).double(), 4, O.down_pad(kern.shape[0], 4))
            self.plan.set_downsampler(torch.from_numpy(kern).float(), 4, self.down[2])
            th, tw = de.down_out_size(H, kern.shape[0], 4, self.down[2]), de.down_out_size(W, kern.shape[0], 4, self.down[2])
        else:
            th, tw = H, W
        self.target = torch.rand(1, cfg.out_channels, th, tw, generator=g).cuda()
        if task == "inpaint":
            self.mask = (torch.rand(1, 1, H, W, generator=g) > 0.3).float().cuda()
        self.params = [p.cuda().contiguous() for p in params_for(cfg, 3)]
        self.grads = [torch.zeros_like(p) for p in self.params]
        self.plan.bind(self.params, self.grads)
        for p, gb in zip(self.params, self.grads):
            p.grad = gb
        self.adam = de.FusedAdam(self.params, lr=lr)
        self.adam._bind(self.grads)
        self.out = torch.empty(1, cfg.out_channels, H, W, device="cuda")

    def check_pin(self, tag, offset):
        """the padded level-0 input is pad(dip_noise_perturb(offset)) bit for bit, with exact zeros in the stored depth's
        channels after the real ones"""
        import dip_engine as de
        zn = torch.empty_like(self.z0)
        de.check(de.lib().dip_noise_perturb(self.z0.data_ptr(), zn.data_ptr(), SIGMA, SEED, offset, self.z0.numel(), None))
        torch.cuda.synchronize()
        want = SR.padding(self.cfg)[0](SR.hwc(zn.double()))
        pin = self.plan.buffer("L0.Pin")
        c = self.cfg.in_channels
        assert pin.shape[-1] == SR.stored_depth(self.cfg, 0)
        assert torch.equal(pin[..., c:], torch.zeros_like(pin[..., c:])), "[%s] stored-depth channels not zero" % tag
        assert torch.equal(pin[..., :c].double(), want), "[%s] L0.Pin != pad(noise stream %d): max |diff| %.3g" % (
            tag, offset, (pin[..., :c].double() - want).abs().max().item())

    def check_stages(self, tag, used, delta=None):
        """every stage and gradient of the last iteration, from the engine's buffers, at parameters `used` (known within
        delta).  The loss / downsampler gradient is checked through the L0.dRaw_v composite, from the output and the
        target; the noisy padded input is taken as given."""
        o = self.out.double().cpu().requires_grad_(True)
        lo = o if self.down is None else O.downsample(o, *self.down)
        loss = O.mse_loss(lo, self.target.double().cpu(), None if self.mask is None else self.mask.double().cpu())
        dout = torch.autograd.grad(loss, o)[0].cuda()
        rd = engine_src(self.plan, self.mode, self.out)
        refs = SR.Refs()
        SR.forward(self.cfg, used, rd, self.mode, refs, delta=delta)
        SR.backward(self.cfg, used, rd, self.mode, refs, dout[0], delta=delta)
        check(tag, self.cfg, self.mode, self.plan, refs, self.grads, self.out)


def run_runner(cfg, H, W, mode, task):
    """one iteration of the device runner (the path bench.py measures) at lr = 0: Adam leaves the parameters bitwise
    unchanged, so the buffers describe one step at known parameters"""
    import dip_engine as de
    r = Runner(cfg, H, W, mode, task, 0.0)
    before = [p.clone() for p in r.params]
    fill_nan(r.plan, cfg.num_scales)
    de.run_iterations(r.plan, r.adam, r.z0, r.target, r.mask, SIGMA, SEED, 1, 0.0, out=r.out)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(before, r.params))
    tag = "runner %s %s %dx%d" % (task, cfg_tag(cfg), H, W)
    r.check_pin(tag, 0)
    r.check_stages(tag, r.params)


@pytest.mark.parametrize("task,kind,H,W,mode", [("denoise", "cs4", 128, 128, "tf32"), ("inpaint", "cs128", 128, 192, "tf32"),
                                                 ("sr", "cs4", 256, 256, "tf32"), ("sr", "cs4", 256, 256, "bf16")])
def test_every_stage_runner(task, kind, H, W, mode):
    run_runner(E.cfg_of(kind), H, W, mode, task)
    print_table()
