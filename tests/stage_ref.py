"""fp64 references of every stage of the engine's training step, in the engine's own layout (test infrastructure).

Every tensor is NHWC without the batch dimension, as `dip_engine.Plan.buffer` returns it: convolution inputs padded as
cfg.pad says (reflection for 'reflection', a zero halo for every other value), the concat in engine order [up (cu
channels) | skip (CS channels)], the concat BatchNorm's gamma / beta rotated to that order (engine channel c is torch
channel (c + CS) % (cu + CS)).  Parameters come in `param_layout` order and torch layout.  The activation behind every
BatchNorm but the concat's is cfg.act_fun.  Everything runs on whatever device the inputs live on, in fp64.

`forward` and `backward` walk the step stage by stage.  Each stage reads its inputs through `src(name)` and records
its reference output (and a per-element tolerance) in a `Refs`.  With `src` = the engine's buffers this is teacher
forcing: every stage is checked from the engine's own inputs, so no error carries over from earlier stages.  With `src`
= the references themselves the stages compose to the whole network (tests/test_stage_ref_cpu.py checks that
composition against the oracle's autograd).

Tolerances (DESIGN.md section 4, "P1 stage"):
  * convolutions: |got - ref| <= 2 (e_op + n 2^-23) M + 2^-23 |bias|, M = the same convolution of |input| and |weight|,
    n = the terms summed per element, e_op = 2^-9 for tf32 (raw fp32 bits are fed to wgmma, each operand keeps 10
    mantissa bits), 0 for fp32 and for bf16 (whose operands the reference reads already rounded);
  * memory-bound stages (fp32 arithmetic in every mode): |got - ref| <= 1e-5 |ref| + 3e-5 s_c, s_c = the reference's RMS
    over channel c; reductions (BatchNorm gamma / beta, head) 1e-5 of the sum of the absolute terms;
  * LeakyReLU boundary: an element whose fp64 pre-activation y lies within 1e-5 (RMS_c(y) + |shift_c| + |mean_c scale_c|)
    of zero may take either slope in fp32 (the kernels evaluate fma(x, scale, shift) in fp32, whose rounding scales with
    all three terms); it is excluded from the elementwise backward checks, and 0.8 |term| of it is added to the tolerance
    of every reduction it enters;
  * act_fun 'Swish', 'ELU', 'none' (models/common.py:76-92): no jump in the first derivative, so no element is excluded
    and the reductions get no flip term.  Instead the kernels evaluate f'(y) in fp32, at the fp32 pre-activation
    fma(x, scale, shift), an error that LeakyReLU, exact off its band, never makes.  It enters dz = g f'(y) like a
    gradient computed on the fly (Bn.backward's `gtol`, propagated the same way):
      |g| (F2 dy + 8 2^-23 (1 + |y|)),  dy = 2 2^-23 (|x scale| + |shift| + |mean scale|),  F2 = sup |f''|
    (dy bounds the rounding of the fp32 pre-activation, the second term that of the fp32 evaluation of f').  It matters
    where the BatchNorm backward cancels: at the deepest level of a 64 x 96 'avg' network a channel has 6 pixels, and
    dx = scale (dz - mean(dz) - xhat mean(dz xhat)) keeps only a small part of dz.  'none' has f' = 1 exactly;
  * parameters reconstructed with an uncertainty (`delta`, param_layout order: |reconstructed - true| <= delta): every
    convolution that multiplies a parameter adds conv(|input|, delta_w) + delta_b to its tolerance (conv_transpose for
    the input gradients); in bf16 mode a tensor-core convolution multiplies bf16(x), whose uncertainty is
    bf16(x + delta) - bf16(x - delta).
The elementwise convolution bound is a worst case and does not tell the precision modes apart (a tf32 product passes
it in fp32 mode), so every convolution output and weight gradient also has a relative Frobenius bound for the mode its
kernel runs in (FROB_TOL): 2e-6 exact fp32, 2e-3 tf32, 3e-5 bf16 operands with fp32 accumulation.
"""
import torch
import torch.nn.functional as F

from oracle import dip_oracle as O

EPS = 1e-5
SLOPE = 0.2
U23 = 2.0 ** -23
E_OP = {"fp64": 0.0, "fp32": 0.0, "tf32": 2.0 ** -9, "bf16": 0.0}
MEM_REL, MEM_ABS = 1e-5, 3e-5
RED_REL = 1e-5
FLIP_BAND = 1e-5
FROB_TOL = {"fp64": 1e-12, "fp32": 2e-6, "tf32": 2e-3, "bf16": 3e-5}


def _swish_grad(y):
    s = torch.sigmoid(y)
    return s * (1 + y * (1 - s))


# the activations other than LeakyReLU: f, f' and sup |f''|
FWD = {k: O.ACTIVATIONS[k] for k in ("Swish", "ELU", "none")}
GRAD = {"Swish": _swish_grad, "ELU": lambda y: torch.where(y > 0, torch.ones_like(y), torch.exp(y)),
        "none": torch.ones_like}
F2 = {"Swish": 0.5, "ELU": 1.0, "none": 0.0}


# ------------------------------------------------------------------------------------------------ layout helpers
def nchw(x):
    return x.permute(2, 0, 1).unsqueeze(0)


def hwc(x):
    return x[0].permute(1, 2, 0)


def reflect_pad(x):
    return hwc(F.pad(nchw(x), (1, 1, 1, 1), mode="reflect"))


def _adjoint(fn, x_shape, g):
    x = torch.zeros(x_shape, dtype=g.dtype, device=g.device, requires_grad=True)
    with torch.enable_grad():
        return torch.autograd.grad(fn(x), x, g)[0]


def fold(gp):
    """adjoint of reflect_pad: padded [(H+2)][(W+2)][C] -> [H][W][C]"""
    return _adjoint(reflect_pad, (gp.shape[0] - 2, gp.shape[1] - 2, gp.shape[2]), gp)


def zero_pad(x):
    """Conv2d(padding=1) in the engine's layout: [H][W][C] -> [(H+2)][(W+2)][C] with a zero halo"""
    return hwc(F.pad(nchw(x), (1, 1, 1, 1)))


def zero_fold(gp):
    """adjoint of zero_pad: the interior of the padded gradient (the halo's gradient is dropped)"""
    return gp[1:-1, 1:-1]


def padding(cfg):
    """(pad, its adjoint) of cfg's 3x3 conv inputs: reflection for pad='reflection', zeros for every other value
    (models/common.py:114-120)"""
    return (reflect_pad, fold) if cfg.pad == "reflection" else (zero_pad, zero_fold)


def upsample(x, bilinear):
    if bilinear:
        return hwc(F.interpolate(nchw(x), scale_factor=2, mode="bilinear", align_corners=False))
    return hwc(F.interpolate(nchw(x), scale_factor=2, mode="nearest"))


def upsample_adj(d, bilinear):
    return _adjoint(lambda x: upsample(x, bilinear), (d.shape[0] // 2, d.shape[1] // 2, d.shape[2]), d)


def chan_rms(x):
    return x.reshape(-1, x.shape[-1]).pow(2).mean(0).sqrt()


def mem_tol(ref):
    return MEM_REL * ref.abs() + MEM_ABS * chan_rms(ref)


def bf16(x):
    return x.to(torch.bfloat16).double()


def rot_param(p, cs):
    """torch-order per-channel parameter of the concat BN -> engine order [up | skip]"""
    return torch.roll(p, -cs) if cs else p


# ------------------------------------------------------------------------------------------------ stages
def conv(x, w, b, stride, mode, unc=None):
    """x: conv input [rows][cols][C] (padded for 3x3) in torch channel order, w OIHW -> (y [h][w][N], tol).
    unc: the (weight, bias) uncertainty of _Reader.unc, or None"""
    X, w = nchw(x.double()), w.double()
    y = F.conv2d(X, w, None if b is None else b.double(), stride=stride)
    m = F.conv2d(X.abs(), w.abs(), None, stride=stride)
    n = w.shape[1] * w.shape[2] * w.shape[3]
    tol = 2 * (E_OP[mode] + n * U23) * m
    if b is not None:
        tol = tol + U23 * b.double().abs().view(1, -1, 1, 1)
    if unc is not None:
        tol = tol + F.conv2d(nchw(x.double().abs()), unc[0], unc[1], stride=stride)
    return hwc(y), hwc(tol)


def conv_dgrad(dy, w, stride, mode, unc=None):
    """input gradient of conv(): dy [h][w][N] -> [rows][cols][C] (the padded extent; stride 2: the last row and column
    of the padded input get no gradient and are returned as 0)"""
    D, w = nchw(dy.double()), w.double()
    g = F.conv_transpose2d(D, w, stride=stride)
    m = F.conv_transpose2d(D.abs(), w.abs(), stride=stride)
    n = w.shape[0] * w.shape[2] * w.shape[3]
    tol = 2 * (E_OP[mode] + n * U23) * m
    if unc is not None:
        tol = tol + F.conv_transpose2d(nchw(dy.double().abs()), unc[0], stride=stride)
    if stride == 2:
        g, tol = F.pad(g, (0, 1, 0, 1)), F.pad(tol, (0, 1, 0, 1))
    return hwc(g), hwc(tol)


def conv_wgrad(x, dy, wshape, stride, mode):
    X, D = nchw(x.double()), nchw(dy.double())
    g = torch.nn.grad.conv2d_weight(X, wshape, D, stride=stride)
    m = torch.nn.grad.conv2d_weight(X.abs(), wshape, D.abs(), stride=stride)
    n = dy.shape[0] * dy.shape[1]
    return g, 2 * (E_OP[mode] + n * U23) * m


class Bn:
    """BatchNorm (training mode, biased variance) of raw [..][C] with engine-order gamma / beta, in fp64, followed by the
    activation `kind` (models.skip's act_fun)"""

    def __init__(self, raw, g, b, kind="LeakyReLU"):
        self.shape, self.kind = raw.shape, kind
        x = raw.double().reshape(-1, raw.shape[-1])
        self.n = x.shape[0]
        mean = x.mean(0)
        self.rstd = 1.0 / ((x - mean).pow(2).mean(0) + EPS).sqrt()
        self.scale = g.double() * self.rstd
        shift = b.double() - mean * self.scale
        self.xhat = (x - mean) * self.rstd
        self.y = x * self.scale + shift
        if kind == "LeakyReLU":
            # elements whose pre-activation may round to the other side of zero in fp32 (the kernels evaluate
            # fma(x, scale, shift) in fp32: its rounding scales with |shift| and |mean * scale| as well)
            band = FLIP_BAND * (chan_rms(self.y) + shift.abs() + (mean * self.scale).abs())
            self.amb = self.y.abs() <= band
        else:   # the fp32 derivative's error per unit of incoming gradient (module docstring)
            dy = 2 * U23 * ((x * self.scale).abs() + shift.abs() + (mean * self.scale).abs())
            self.dact = 0.0 if kind == "none" else F2[kind] * dy + 8 * U23 * (1 + self.y.abs())

    def out(self, act=True):
        if not act:
            y = self.y
        elif self.kind == "LeakyReLU":
            y = torch.where(self.y > 0, self.y, SLOPE * self.y)
        else:
            y = FWD[self.kind](self.y)
        return y.reshape(self.shape)

    def backward(self, gout, act=True, gtol=None):
        """gout = dL/d(output), gtol = its tolerance where the engine computes it on the fly (fold + skip-conv term)
        -> dict(dx, dgamma, dbeta (engine order), their tolerances, the excluded elements and their share)"""
        go = gout.double().reshape(-1, self.shape[-1])
        xh = self.xhat
        gt = torch.zeros_like(go) if gtol is None else gtol.double().reshape(-1, self.shape[-1])
        leaky = act and self.kind == "LeakyReLU"
        if not act:
            dz, flip = go, torch.zeros_like(go)
        elif leaky:
            dz = torch.where(self.y > 0, go, SLOPE * go)
            flip = (1 - SLOPE) * go.abs() * self.amb
        else:
            d = GRAD[self.kind](self.y)
            dz, flip = go * d, None
            gt = gt * d.abs() + go.abs() * self.dact
        m1, m2 = dz.mean(0), (dz * xh).mean(0)
        dx = self.scale * (dz - m1 - xh * m2)
        fg = gt if flip is None else flip + gt
        f1, f2 = fg.sum(0), (fg * xh.abs()).sum(0)
        tol_dx = mem_tol(dx) + self.scale.abs() * (gt + (f1 + xh.abs() * f2) / self.n)
        excl = self.amb if leaky else torch.zeros_like(go, dtype=torch.bool)
        return dict(dx=dx.reshape(self.shape), tol_dx=tol_dx.reshape(self.shape), excl=excl.reshape(self.shape),
                    dbeta=dz.sum(0), tol_dbeta=RED_REL * dz.abs().sum(0) + f1,
                    dgamma=(dz * xh).sum(0), tol_dgamma=RED_REL * (dz * xh).abs().sum(0) + f2,
                    excl_frac=excl.double().mean().item())


class CatBn(Bn):
    """The concat BatchNorm's backward as the engine evaluates it: xhat = (y - beta) / gamma recovered from the stored,
    padded output P_cat, rstd from the statistics of the pre-BN concat (recorded by forward())"""

    def __init__(self, pcat, g, b, rstd):
        y = pcat.double()[1:-1, 1:-1]
        self.shape = y.shape
        self.n = y.shape[0] * y.shape[1]
        self.rstd = rstd
        self.scale = g.double() * rstd
        self.xhat = ((y - b.double()) / g.double()).reshape(-1, y.shape[-1])


class Refs:
    """name -> (reference, tolerance, excluded elements or None).  Parameter gradients are recorded as 'grad:<name>',
    the share of excluded elements of every LeakyReLU backward in `excl`, values that later stages need in `aux`."""

    def __init__(self):
        self.d, self.excl, self.aux = {}, {}, {}
        self.conv = {}   # convolution outputs / weight gradients -> the precision mode they run at (FROB_TOL key)

    def put(self, name, ref, tol, excl=None):
        self.d[name] = (ref, tol, excl)

    def put_conv(self, name, mode, ref, tol):
        self.put(name, ref, tol)
        self.conv[name] = mode

    def put_bwd(self, name, res):
        self.put(name, res["dx"], res["tol_dx"], res["excl"])
        self.excl[name] = (res["excl_frac"], res["dx"].numel())

    def __getitem__(self, name):
        return self.d[name][0]

    def __contains__(self, name):
        return name in self.d


def _params(cfg, params):
    return {n: p.detach().double() for (n, _), p in zip(O.param_layout(cfg), params)}


def _twin(name):
    """bf16 twin of a buffer: L0.Pin -> L0.Pin16, L0.P_d1 -> L0.P_d1_16"""
    return name + ("_16" if name[-1].isdigit() else "16")


class _Reader:
    """src(name) in fp64; .op(name) is the operand a tensor-core convolution reads (its bf16 twin in bf16 mode); .w(name)
    is a tensor-core convolution's weight as the kernel multiplies it (bf16 mode: rounded to bf16); .unc(layer) the
    uncertainty of a convolution's parameters (D: name -> delta, or None for exact parameters)"""

    def __init__(self, src, P, mode, D=None):
        self.src, self.P, self.mode, self.D = src, P, mode, D

    def __call__(self, name):
        return self.src(name).double()

    def op(self, name, c=None):
        t = self.src(_twin(name) if self.mode == "bf16" else name).double()
        return t if c is None else t[..., :c]

    def w(self, name):
        return bf16(self.P[name]) if self.mode == "bf16" else self.P[name]

    def unc(self, layer, tc=True):
        """(weight, bias) uncertainty of conv `layer` as its kernel multiplies them (tc: a tensor-core convolution, which
        multiplies bf16(x) in bf16 mode), or None"""
        if self.D is None:
            return None
        dw, db = self.D[layer + ".w"], self.D[layer + ".b"]
        if tc and self.mode == "bf16":
            x = self.P[layer + ".w"]
            dw = bf16(x + dw) - bf16(x - dw)
        return dw, db


def is_dead_bias(name):
    """a conv bias in front of a BatchNorm: its gradient is 0 in exact arithmetic"""
    return name.endswith(".b") and "_bn" not in name and not name.startswith("head")


def stored_depth(cfg, l):
    """depth of the engine's level-l input: level 0 rounds the input depth up to a power of two >= 4 (zero channels)"""
    if l > 0:
        return cfg.nd(l - 1)
    c = 4
    while c < cfg.in_channels:
        c *= 2
    return c


def _up_mode(cfg, l):
    m = cfg.upsample_mode if isinstance(cfg.upsample_mode, str) else cfg.upsample_mode[l]
    return m == "bilinear"


def forward(cfg, params, src, mode, refs, z=None, noise=None, sigma=0.0, delta=None):
    """References of every forward stage and of the network output ('out', torch layout K x H x W).
    z / noise: torch-layout 1 x C x H x W inputs of the level-0 input transform (None: the padded input L0.Pin is taken
    as given, as for the runner, whose noise is generated on the device).  delta: the parameters' uncertainty, in
    param_layout order (None: exact)."""
    P = _params(cfg, params)
    rd = _Reader(src, P, mode, None if delta is None else _params(cfg, delta))
    pad, act = padding(cfg)[0], cfg.act_fun
    L = cfg.num_scales
    if z is not None:
        x = z.double() if noise is None else z.double() + sigma * noise.double()
        x = F.pad(hwc(x), (0, stored_depth(cfg, 0) - x.shape[1]))   # the stored depth's extra channels are zeros
        refs.put("L0.Pin", pad(x), mem_tol(pad(x)))
    for l in range(L):
        pf = "L%d." % l
        cs, cin = cfg.ns(l), (cfg.in_channels if l == 0 else cfg.nd(l - 1))
        if cs == 4:   # skinny CUDA-core conv on the fp32 input
            refs.put_conv(pf + "raw_s", "fp32", *conv(rd(pf + "Pin")[1:-1, 1:-1, :cin], P[pf + "skip.w"], P[pf + "skip.b"], 1, "fp32",
                                                   rd.unc(pf + "skip", tc=False)))
        elif cs == 128:
            refs.put_conv(pf + "raw_s", mode, *conv(rd.op(pf + "Pin", cin)[1:-1, 1:-1], rd.w(pf + "skip.w"), P[pf + "skip.b"], 1, mode,
                                                rd.unc(pf + "skip")))
        if cfg.downsample_mode == "avg":   # stride-1 conv + AvgPool2d(2, 2)
            refs.put_conv(pf + "rawF", mode, *conv(rd.op(pf + "Pin", cin), rd.w(pf + "d1.w"), P[pf + "d1.b"], 1, mode, rd.unc(pf + "d1")))
            y = hwc(F.avg_pool2d(nchw(rd(pf + "rawF")), 2, 2))
            refs.put(pf + "raw_d1", y, mem_tol(y))
        else:
            refs.put_conv(pf + "raw_d1", mode, *conv(rd.op(pf + "Pin", cin), rd.w(pf + "d1.w"), P[pf + "d1.b"], 2, mode, rd.unc(pf + "d1")))
        y = pad(Bn(rd(pf + "raw_d1"), P[pf + "d1_bn.g"], P[pf + "d1_bn.b"], act).out())
        refs.put(pf + "P_d1", y, mem_tol(y))
        refs.put_conv(pf + "raw_d2", mode, *conv(rd.op(pf + "P_d1"), rd.w(pf + "d2.w"), P[pf + "d2.b"], 1, mode, rd.unc(pf + "d2")))
        y = Bn(rd(pf + "raw_d2"), P[pf + "d2_bn.g"], P[pf + "d2_bn.b"], act).out()
        y = y if l == L - 1 else pad(y)
        refs.put(pf + "P_d2", y, mem_tol(y))
    for l in reversed(range(L)):
        pf = "L%d." % l
        cs, nu = cfg.ns(l), cfg.nu(l)
        low = rd(pf + "P_d2") if l == L - 1 else rd("L%d.U" % (l + 1))
        parts = [upsample(low, _up_mode(cfg, l))]
        if cs:
            parts.append(Bn(rd(pf + "raw_s"), P[pf + "skip_bn.g"], P[pf + "skip_bn.b"], act).out())
        bn = Bn(torch.cat(parts, -1), rot_param(P[pf + "cat_bn.g"], cs), rot_param(P[pf + "cat_bn.b"], cs))
        y = pad(bn.out(act=False))
        refs.put(pf + "P_cat", y, mem_tol(y))
        refs.aux[pf + "cat_rstd"] = bn.rstd
        x = torch.roll(rd.op(pf + "P_cat"), cs, -1)   # torch channel order [skip | up]
        refs.put_conv(pf + "raw_u", mode, *conv(x, rd.w(pf + "up.w"), P[pf + "up.b"], 1, mode, rd.unc(pf + "up")))
        y = Bn(rd(pf + "raw_u"), P[pf + "up_bn.g"], P[pf + "up_bn.b"], act).out()
        refs.put(pf + "A_u", y, mem_tol(y))
        refs.put_conv(pf + "raw_v", mode, *conv(rd.op(pf + "A_u"), rd.w(pf + "c11.w"), P[pf + "c11.b"], 1, mode, rd.unc(pf + "c11")))
        u = Bn(rd(pf + "raw_v"), P[pf + "c11_bn.g"], P[pf + "c11_bn.b"], act).out()
        if l > 0 or nu != 128:
            refs.put(pf + "U", u, mem_tol(u))
        if l == 0:   # RGB head (+ sigmoid): a skinny conv over U where U is materialised, else fused into the BN of raw_v
            if nu != 128:
                u = rd(pf + "U")
            terms = torch.einsum("hwc,kc->khwc", u, P["head.w"][:, :, 0, 0])
            logit = terms.sum(-1) + P["head.b"].view(-1, 1, 1)
            tol = RED_REL * (terms.abs().sum(-1) + P["head.b"].abs().view(-1, 1, 1))
            if cfg.need_sigmoid:
                refs.put("out", torch.sigmoid(logit), 0.25 * tol)
            else:
                refs.put("out", logit, tol)


def head_logit_grad(dout, out, sigmoid):
    """dL/d(logit) [K][H][W] from dL/d(out) and the network output"""
    dout, out = dout.double(), out.double()
    return dout * out * (1 - out) if sigmoid else dout


def backward(cfg, params, src, mode, refs, dout, input_grad=False, delta=None):
    """References of every backward stage and of every parameter gradient ('grad:<param_layout name>', torch layout).
    dout: dL/d(out) [K][H][W]; 'out' is read through src.  forward() must have filled `refs` first (concat statistics).
    delta: as for forward()."""
    P = _params(cfg, params)
    rd = _Reader(src, P, mode, None if delta is None else _params(cfg, delta))
    fold, act = padding(cfg)[1], cfg.act_fun
    L = cfg.num_scales
    avg = cfg.downsample_mode == "avg"

    def bn_grads(pf, bn, res, cs=0, bias=None):
        refs.put("grad:" + pf + bn + ".g", torch.roll(res["dgamma"], cs), torch.roll(res["tol_dgamma"], cs))
        refs.put("grad:" + pf + bn + ".b", torch.roll(res["dbeta"], cs), torch.roll(res["tol_dbeta"], cs))
        if bias is not None:   # conv bias in front of a BatchNorm: its gradient is 0 in exact arithmetic
            dx = res["dx"].reshape(-1, res["dx"].shape[-1])
            refs.put("grad:" + pf + bias + ".b", torch.zeros_like(dx[0]), RED_REL * dx.abs().sum(0))

    for l in range(L):
        pf = "L%d." % l
        cs, cu, nu = cfg.ns(l), cfg.cu(l), cfg.nu(l)
        cin = cfg.in_channels if l == 0 else cfg.nd(l - 1)
        bnv = Bn(rd(pf + "raw_v"), P[pf + "c11_bn.g"], P[pf + "c11_bn.b"], act)
        if l == 0:   # RGB head adjoint fused into the BN backward (GradSrc kind 3), and the head's own gradients
            dl = head_logit_grad(dout.to(bnv.y.device), rd("out"), cfg.need_sigmoid)
            wh = P["head.w"][:, :, 0, 0]
            gsrc = torch.einsum("khw,kc->hwc", dl, wh)
            terms = torch.einsum("khw,hwc->kchw", dl, bnv.out())
            refs.put("grad:head.w", terms.sum((2, 3))[..., None, None], (RED_REL * terms.abs().sum((2, 3)))[..., None, None])
            refs.put("grad:head.b", dl.sum((1, 2)), RED_REL * dl.abs().sum((1, 2)))
        else:
            gsrc = rd("L%d.dUp" % (l - 1))
        res = bnv.backward(gsrc)
        refs.put_bwd(pf + "dRaw_v", res)
        bn_grads(pf, "c11_bn", res, bias="c11")
        dy = rd.op(pf + "dRaw_v")
        refs.put_conv(pf + "dA_u", mode, *conv_dgrad(dy, rd.w(pf + "c11.w"), 1, mode, rd.unc(pf + "c11")))
        refs.put_conv("grad:" + pf + "c11.w", mode, *conv_wgrad(rd.op(pf + "A_u"), dy, (nu, nu, 1, 1), 1, mode))
        res = Bn(rd(pf + "raw_u"), P[pf + "up_bn.g"], P[pf + "up_bn.b"], act).backward(rd(pf + "dA_u"))
        refs.put_bwd(pf + "dRaw_u", res)
        bn_grads(pf, "up_bn", res, bias="up")
        dy = rd.op(pf + "dRaw_u")
        g, t = conv_dgrad(dy, rd.w(pf + "up.w"), 1, mode, rd.unc(pf + "up"))
        refs.put_conv(pf + "dP_cat", mode, torch.roll(g, -cs, -1), torch.roll(t, -cs, -1))
        refs.put_conv("grad:" + pf + "up.w", mode, *conv_wgrad(torch.roll(rd.op(pf + "P_cat"), cs, -1), dy, (nu, cu + cs, 3, 3), 1, mode))
        gc, bc = rot_param(P[pf + "cat_bn.g"], cs), rot_param(P[pf + "cat_bn.b"], cs)
        res = CatBn(rd(pf + "P_cat"), gc, bc, refs.aux[pf + "cat_rstd"]).backward(fold(rd(pf + "dP_cat")), act=False)
        refs.put(pf + "dCat", res["dx"], res["tol_dx"])
        bn_grads(pf, "cat_bn", res, cs)
        dcat = rd(pf + "dCat")
        g = upsample_adj(dcat[..., :cu], _up_mode(cfg, l))
        refs.put(pf + "dUp", g, mem_tol(g))
        if cs:
            res = Bn(rd(pf + "raw_s"), P[pf + "skip_bn.g"], P[pf + "skip_bn.b"], act).backward(dcat[..., cu:])
            refs.put_bwd(pf + "dRaw_s", res)
            bn_grads(pf, "skip_bn", res, bias="skip")
            md = mode if cs == 128 else "fp32"   # the 4-channel skip conv runs on the CUDA cores in fp32
            pin = (rd.op(pf + "Pin", cin) if cs == 128 else rd(pf + "Pin")[..., :cin])[1:-1, 1:-1]
            dys = rd.op(pf + "dRaw_s") if cs == 128 else rd(pf + "dRaw_s")
            refs.put_conv("grad:" + pf + "skip.w", md, *conv_wgrad(pin, dys, (cs, cin, 1, 1), 1, md))
            if l > 0 and cs == 128 or l == 0 and input_grad:
                g, t = conv_dgrad(dys, rd.w(pf + "skip.w") if cs == 128 else P[pf + "skip.w"], 1, md,
                                  rd.unc(pf + "skip", tc=cs == 128))
                pad = (0, stored_depth(cfg, l) - cin)
                refs.put_conv(pf + "dS", md, F.pad(g, pad), F.pad(t, pad))
    for l in reversed(range(L)):
        pf = "L%d." % l
        nd, cin = cfg.nd(l), (cfg.in_channels if l == 0 else cfg.nd(l - 1))
        if l == L - 1:
            g, gtol = rd(pf + "dUp"), None
        else:   # fold of the next level's padded input gradient + the input gradient of its skip conv
            n = "L%d." % (l + 1)
            g = fold(rd(n + "dPin"))
            gtol = mem_tol(g)
            if cfg.ns(l + 1) == 4:
                t = torch.einsum("hwn,nc->hwnc", rd(n + "dRaw_s"), P[n + "skip.w"][:, :, 0, 0])
                g, gtol = g + t.sum(2), gtol + RED_REL * t.abs().sum(2)
            elif cfg.ns(l + 1) == 128:
                g, gtol = g + rd(n + "dS"), gtol + mem_tol(rd(n + "dS"))
        res = Bn(rd(pf + "raw_d2"), P[pf + "d2_bn.g"], P[pf + "d2_bn.b"], act).backward(g, gtol=gtol)
        refs.put_bwd(pf + "dRaw_d2", res)
        bn_grads(pf, "d2_bn", res, bias="d2")
        dy = rd.op(pf + "dRaw_d2")
        refs.put_conv(pf + "dP_d1", mode, *conv_dgrad(dy, rd.w(pf + "d2.w"), 1, mode, rd.unc(pf + "d2")))
        refs.put_conv("grad:" + pf + "d2.w", mode, *conv_wgrad(rd.op(pf + "P_d1"), dy, (nd, nd, 3, 3), 1, mode))
        res = Bn(rd(pf + "raw_d1"), P[pf + "d1_bn.g"], P[pf + "d1_bn.b"], act).backward(fold(rd(pf + "dP_d1")))
        refs.put_bwd(pf + "dRaw_d1", res)
        bn_grads(pf, "d1_bn", res, bias="d1")
        if avg:   # adjoint of AvgPool2d(2, 2): the conv's dY at full resolution
            g = 0.25 * rd(pf + "dRaw_d1").repeat_interleave(2, 0).repeat_interleave(2, 1)
            refs.put(pf + "dRawF", g, mem_tol(g))
            dy, stride = rd.op(pf + "dRawF"), 1
        else:
            dy, stride = rd.op(pf + "dRaw_d1"), 2
        if l > 0 or input_grad:   # (level 0: the real input depth; the stored depth's extra channels get no gradient)
            refs.put_conv(pf + "dPin", mode, *conv_dgrad(dy, rd.w(pf + "d1.w"), stride, mode, rd.unc(pf + "d1")))
        refs.put_conv("grad:" + pf + "d1.w", mode, *conv_wgrad(rd.op(pf + "Pin", cin), dy, (nd, cin, 3, 3), stride, mode))
    if input_grad:   # dL/d(net input), torch layout 1 x C x H x W
        g = fold(rd("L0.dPin"))[..., :cfg.in_channels]
        if cfg.ns(0):
            g = g + rd("L0.dS")[..., :cfg.in_channels]
        refs.put("dz", nchw(g), nchw(mem_tol(g)))


def random_affine(cfg, params, seed):
    """Parameters away from init: every BatchNorm gamma U(0.5, 1.5), every beta and conv bias U(-0.5, 0.5) (a concat BN
    gets different values for its skip and up channels, so a rotation error shows); conv weights are kept."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for (name, shape), p in zip(O.param_layout(cfg), params):
        p = p.detach().clone()
        if name.endswith("_bn.g"):
            p.copy_(0.5 + torch.rand(shape, generator=g, dtype=torch.float64))
        elif name.endswith(".b"):
            p.copy_(torch.rand(shape, generator=g, dtype=torch.float64) - 0.5)
        out.append(p)
    return out
