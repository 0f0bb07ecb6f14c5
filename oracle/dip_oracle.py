"""CPU oracle for the deep-image-prior hot path -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this module;
the product path (deep-image-prior_b200/) never does.

What it is: a self-contained restatement, on torch-CPU functional ops, of what the reference executes per iteration
(the reference's arithmetic lives in its third-party dependency PyTorch -- pinned `pytorch=0.4` in environment.yml:13,
installed here: torch 2.11 -- so the oracle restates the reference's *graph* on the same dependency):

  * skip-network forward            models/skip.py:41-100 + models/common.py:11-124 (Concat, conv, bn, act)
  * parameter initialisation order  models/skip.py:45-98 (construction order = RNG draw order)
  * loss                            torch.nn.MSELoss, denoising.ipynb c8:50, c10:23; masked: inpainting.ipynb c17:17
  * optimiser                       torch.optim.Adam defaults, utils/common_utils.py:225-230
  * input perturbation              denoising.ipynb c10:12-13
  * get_noise                       utils/common_utils.py:127-153
  * Downsampler / get_kernel        models/downsampler.py:5-135 (super-resolution operator, super-resolution.ipynb c10:8)

Pinning: the reference has NO golden vectors / tests (SURVEY.md section 4, 8c).  The oracle is pinned instead against
outputs of the reference itself, generated in the build container by tests/golden/make_golden.py (which imports
/root/reference) and committed as tests/golden/*.npz; tests/test_oracle.py checks oracle == golden, and
oracle == live reference whenever /root/reference is present.
"""
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F


class SkipConfig:
    """Arguments of models.skip() that matter for the BASELINE configs (models/skip.py:5-11)."""

    def __init__(self, in_channels=32, out_channels=3, num_scales=5, channels=128, skip_channels=4,
                 upsample_mode="bilinear", need_sigmoid=True):
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.num_scales = num_scales
        self.channels = channels
        self.skip_channels = skip_channels
        self.upsample_mode = upsample_mode
        self.need_sigmoid = need_sigmoid

    # per-scale widths (models/skip.py:6-7): `channels` / `skip_channels` may be one int for every scale or a sequence
    # (num_channels_down = num_channels_up = channels unless channels_up is set: denoising.ipynb c8:17-23 "snail")
    channels_up = None
    # in-net downsampling of the first down conv (models/common.py:101-113): 'stride' (stride-2 conv) or 'avg'
    # (stride-1 conv + nn.AvgPool2d(2, 2): restoration.ipynb c7:28-36 kate)
    downsample_mode = "stride"
    # padding of every conv with k > 1 (models/common.py:114-120): 'reflection' is nn.ReflectionPad2d(k // 2), any other
    # value Conv2d(padding=k // 2), i.e. zeros (models.skip's own default is pad='zero')
    pad = "reflection"
    # activation behind every BatchNorm but the concat's (models/common.py:76-92): a key of ACTIVATIONS
    act_fun = "LeakyReLU"

    def nd(self, l):
        return self.channels[l] if isinstance(self.channels, (list, tuple)) else self.channels

    def nu(self, l):
        if self.channels_up is not None:
            return self.channels_up[l]
        return self.nd(l)

    def ns(self, l):
        return self.skip_channels[l] if isinstance(self.skip_channels, (list, tuple)) else self.skip_channels

    def cu(self, l):
        """depth of the tensor upsampled into scale l's concat (models/skip.py:48-55)"""
        return self.nu(l + 1) if l < self.num_scales - 1 else self.nd(l)


def param_layout(cfg):
    """[(name, shape)] in net.parameters() order of the reference (depth-first over the module tree)."""
    L = cfg.num_scales
    pre, post = [], []
    for l in range(L):
        C, S = cfg.nd(l), cfg.ns(l)
        cin = cfg.in_channels if l == 0 else cfg.nd(l - 1)
        sk = [("L%d.skip.w" % l, (S, cin, 1, 1)), ("L%d.skip.b" % l, (S,)),
              ("L%d.skip_bn.g" % l, (S,)), ("L%d.skip_bn.b" % l, (S,))] if S > 0 else []   # num_channels_skip = 0: no skip branch
        pre.append(sk + [
                    ("L%d.d1.w" % l, (C, cin, 3, 3)), ("L%d.d1.b" % l, (C,)),
                    ("L%d.d1_bn.g" % l, (C,)), ("L%d.d1_bn.b" % l, (C,)),
                    ("L%d.d2.w" % l, (C, C, 3, 3)), ("L%d.d2.b" % l, (C,)),
                    ("L%d.d2_bn.g" % l, (C,)), ("L%d.d2_bn.b" % l, (C,))])
        U, K = cfg.nu(l), cfg.cu(l) + S
        post.append([("L%d.cat_bn.g" % l, (K,)), ("L%d.cat_bn.b" % l, (K,)),
                     ("L%d.up.w" % l, (U, K, 3, 3)), ("L%d.up.b" % l, (U,)),
                     ("L%d.up_bn.g" % l, (U,)), ("L%d.up_bn.b" % l, (U,)),
                     ("L%d.c11.w" % l, (U, U, 1, 1)), ("L%d.c11.b" % l, (U,)),
                     ("L%d.c11_bn.g" % l, (U,)), ("L%d.c11_bn.b" % l, (U,))])
    out = []
    for l in range(L):
        out += pre[l]
    for l in reversed(range(L)):
        out += post[l]
    out += [("head.w", (cfg.out_channels, cfg.nu(0), 1, 1)), ("head.b", (cfg.out_channels,))]
    return out


def init_params(cfg, seed=None, dtype=torch.float32):
    """Parameters with the reference's initialisation AND RNG draw order (models/skip.py:45-98: per level the convs
    are constructed skip, down1, down2, up3x3, up1x1; levels top-down; head last; BatchNorm draws nothing)."""
    if seed is not None:
        torch.manual_seed(seed)
    L = cfg.num_scales
    vals = {}
    for l in range(L):
        C, U, S = cfg.nd(l), cfg.nu(l), cfg.ns(l)
        cin = cfg.in_channels if l == 0 else cfg.nd(l - 1)
        for name, (o, i, k) in (("skip", (S, cin, 1)), ("d1", (C, cin, 3)), ("d2", (C, C, 3)), ("up", (U, cfg.cu(l) + S, 3)),
                                ("c11", (U, U, 1))):
            if o == 0:
                continue   # models/skip.py:57-60: the skip conv is only constructed (and only draws from the RNG) when it has channels
            m = nn.Conv2d(i, o, k)  # torch default init: kaiming_uniform(a=sqrt(5)) + bias U(+-1/sqrt(fan_in))
            vals["L%d.%s.w" % (l, name)] = m.weight.detach()
            vals["L%d.%s.b" % (l, name)] = m.bias.detach()
    m = nn.Conv2d(cfg.nu(0), cfg.out_channels, 1)
    vals["head.w"], vals["head.b"] = m.weight.detach(), m.bias.detach()
    params = []
    for name, shape in param_layout(cfg):
        if name in vals:
            t = vals[name]
        elif name.endswith(".g"):
            t = torch.ones(shape)
        else:
            t = torch.zeros(shape)
        params.append(t.to(dtype).clone().requires_grad_(True))
    return params


# ---- bf16-operand emulation (the checker of the engine's precision mode 'bf16', BASELINE.json configs[2]) -------------
# The reference has no bf16 path of its own (its GPU path is fp32 / cuDNN-TF32; "bf16" is BASELINE.json's wording for the
# super-resolution configuration).  The engine's definition: every convolution that runs on the tensor cores -- the wide
# convs, 8 or more output channels -- reads its input, its weight and, in the backward pass, the incoming gradient
# ROUNDED TO BF16 (round to nearest even), multiplies exactly and accumulates in fp32; biases, BatchNorm, activations,
# up-sampling, the skinny skip convs, the head, the loss and Adam stay fp32.  `with operand_rounding('bf16'):` makes
# conv2d evaluate exactly that definition on the CPU (in whatever dtype the parameters have, fp64 included).
_OPERAND_ROUND = None
_MIN_TENSOR_CORE_WIDTH = 8   # the skinny skip convs (4 outputs) and the head (<= 4) run in fp32 on the CUDA cores


class operand_rounding:
    def __init__(self, kind):
        assert kind in (None, "bf16")
        self.kind = kind

    def __enter__(self):
        global _OPERAND_ROUND
        self.prev, _OPERAND_ROUND = _OPERAND_ROUND, self.kind

    def __exit__(self, *a):
        global _OPERAND_ROUND
        _OPERAND_ROUND = self.prev


def _round_bf16(t):
    return t.to(torch.bfloat16).to(t.dtype)


class _ConvBf16Operands(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, stride):
        xr, wr = _round_bf16(x), _round_bf16(w)
        ctx.save_for_backward(xr, wr)
        ctx.stride = stride
        return F.conv2d(xr, wr, b, stride=stride)

    @staticmethod
    def backward(ctx, dy):
        xr, wr = ctx.saved_tensors
        dyr = _round_bf16(dy)
        dx = torch.nn.grad.conv2d_input(xr.shape, wr, dyr, stride=ctx.stride)
        dw = torch.nn.grad.conv2d_weight(xr, wr.shape, dyr, stride=ctx.stride)
        return dx, dw, dy.sum((0, 2, 3)), None


def conv2d(x, w, b, stride=1, pad="reflection"):
    k = w.shape[-1]
    if k > 1:   # nn.ReflectionPad2d or Conv2d(padding=k // 2), models/common.py:114-120
        x = F.pad(x, (k // 2,) * 4, mode="reflect" if pad == "reflection" else "constant")
    if _OPERAND_ROUND == "bf16" and w.shape[0] >= _MIN_TENSOR_CORE_WIDTH:
        return _ConvBf16Operands.apply(x, w, b, stride)
    return F.conv2d(x, w, b, stride=stride)


def _bn(x, g, b):
    # nn.BatchNorm2d in training mode (nothing in the reference ever calls .eval()): biased batch variance, eps 1e-5
    return F.batch_norm(x, None, None, g, b, training=True, momentum=0.1, eps=1e-5)


ACTIVATIONS = {"LeakyReLU": lambda x: F.leaky_relu(x, 0.2), "Swish": lambda x: x * torch.sigmoid(x), "ELU": F.elu,
               "none": lambda x: x}   # act(): nn.LeakyReLU(0.2), Swish, nn.ELU(), nn.Sequential()


def activation(x, kind="LeakyReLU"):
    if kind not in ACTIVATIONS:
        raise ValueError("act_fun must be one of %s, not %r" % (", ".join(ACTIVATIONS), kind))
    return ACTIVATIONS[kind](x)


# the earlier names (test_oracle.py calls _conv directly).  skip_forward calls conv2d and activation, so the padding and
# the activation of a network come from its cfg alone, whatever a caller may have rebound these two names to.
_conv, _act = conv2d, activation


def skip_forward(params, z, cfg, tape=None):
    """out = net(z).  params in param_layout() order.  tape (dict) receives named intermediates (for debugging)."""
    P = {name: p for (name, _), p in zip(param_layout(cfg), params)}

    def rec(l, x):
        pre = "L%d." % l
        s = None
        if cfg.ns(l) > 0:
            s = conv2d(x, P[pre + "skip.w"], P[pre + "skip.b"], pad=cfg.pad)
            if tape is not None:
                tape[pre + "raw_s"] = s
            s = activation(_bn(s, P[pre + "skip_bn.g"], P[pre + "skip_bn.b"]), cfg.act_fun)
        if cfg.downsample_mode == "avg":
            d = F.avg_pool2d(conv2d(x, P[pre + "d1.w"], P[pre + "d1.b"], stride=1, pad=cfg.pad), 2, 2)
        else:
            d = conv2d(x, P[pre + "d1.w"], P[pre + "d1.b"], stride=2, pad=cfg.pad)
        if tape is not None:
            tape[pre + "raw_d1"] = d
        d = activation(_bn(d, P[pre + "d1_bn.g"], P[pre + "d1_bn.b"]), cfg.act_fun)
        d = conv2d(d, P[pre + "d2.w"], P[pre + "d2.b"], pad=cfg.pad)
        if tape is not None:
            tape[pre + "raw_d2"] = d
        d = activation(_bn(d, P[pre + "d2_bn.g"], P[pre + "d2_bn.b"]), cfg.act_fun)
        if l < cfg.num_scales - 1:
            d = rec(l + 1, d)
        mode = cfg.upsample_mode if isinstance(cfg.upsample_mode, str) else cfg.upsample_mode[l]   # per scale: skip.py:81
        if mode == "bilinear":
            d = F.interpolate(d, scale_factor=2, mode="bilinear", align_corners=False)
        else:
            d = F.interpolate(d, scale_factor=2, mode="nearest")
        c = torch.cat([s, d], dim=1) if s is not None else d  # Concat: skip channels first (models/common.py:19-39); skip.py:50-53
        if tape is not None:
            tape[pre + "cat"] = c
        c = _bn(c, P[pre + "cat_bn.g"], P[pre + "cat_bn.b"])
        u = conv2d(c, P[pre + "up.w"], P[pre + "up.b"], pad=cfg.pad)
        if tape is not None:
            tape[pre + "raw_u"] = u
        u = activation(_bn(u, P[pre + "up_bn.g"], P[pre + "up_bn.b"]), cfg.act_fun)
        v = conv2d(u, P[pre + "c11.w"], P[pre + "c11.b"], pad=cfg.pad)
        if tape is not None:
            tape[pre + "raw_v"] = v
        v = activation(_bn(v, P[pre + "c11_bn.g"], P[pre + "c11_bn.b"]), cfg.act_fun)
        if tape is not None:
            tape[pre + "U"] = v
        return v

    y = rec(0, z)
    y = F.conv2d(y, P["head.w"], P["head.b"])
    if cfg.need_sigmoid:
        y = torch.sigmoid(y)
    return y


def mse_loss(out, target, mask=None):
    """torch.nn.MSELoss()(out, target) / masked variant mse(out*mask, target*mask) (mean over all C*H*W)."""
    if mask is not None:
        return F.mse_loss(out * mask, target * mask)
    return F.mse_loss(out, target)


def get_noise(input_depth, spatial_size, var=0.1, seed=None):
    """utils/common_utils.py:127-153 with method='noise', noise_type='u'."""
    if seed is not None:
        torch.manual_seed(seed)
    if isinstance(spatial_size, int):
        spatial_size = (spatial_size, spatial_size)
    z = torch.zeros([1, input_depth, spatial_size[0], spatial_size[1]])
    z.uniform_()
    z *= var
    return z


class Adam:
    """torch.optim.Adam defaults (beta 0.9/0.999, eps 1e-8), written out in the order of torch/optim/adam.py."""

    def __init__(self, params, lr):
        self.params, self.lr, self.t = params, lr, 0
        self.m = [torch.zeros_like(p) for p in params]
        self.v = [torch.zeros_like(p) for p in params]

    def step(self, grads):
        self.t += 1
        b1, b2, eps = 0.9, 0.999, 1e-8
        bc1 = 1 - b1 ** self.t
        bc2 = 1 - b2 ** self.t
        with torch.no_grad():
            for p, g, m, v in zip(self.params, grads, self.m, self.v):
                m.lerp_(g, 1 - b1)
                v.mul_(b2).addcmul_(g, g, value=1 - b2)
                denom = (v.sqrt() / math.sqrt(bc2)).add_(eps)
                p.addcdiv_(m, denom, value=-self.lr / bc1)


def down_kernel(factor, kernel_type, phase=0.5, kernel_width=None, support=None, sigma=None):
    """K x K float64 filter of the Downsampler, normalised to sum 1 (models/downsampler.py:73-135, element by element;
    presets lanczos2 / lanczos3 / gauss12 / gauss1sq2 as at models/downsampler.py:14-33)."""
    presets = {"lanczos2": ("lanczos", 2, 4 * factor + 1, None), "lanczos3": ("lanczos", 3, 6 * factor + 1, None),
               "gauss12": ("gauss", None, 7, 0.5), "gauss1sq2": ("gauss", None, 9, 1.0 / math.sqrt(2.0))}
    if kernel_type in presets:
        kernel_type, sup, kernel_width, sig = presets[kernel_type]
        support = sup if sup is not None else support
        sigma = sig if sig is not None else sigma
    n = kernel_width - 1 if (phase == 0.5 and kernel_type != "box") else kernel_width
    k = np.zeros((n, n), dtype=np.float64)
    centre = (kernel_width + 1) / 2.0
    for i in range(1, n + 1):
        for j in range(1, n + 1):
            if kernel_type == "box":
                k[i - 1, j - 1] = 1.0 / (kernel_width * kernel_width)
            elif kernel_type == "gauss":
                di, dj = (i - centre) / 2.0, (j - centre) / 2.0
                k[i - 1, j - 1] = math.exp(-(di * di + dj * dj) / (2 * sigma * sigma)) / (2.0 * math.pi * sigma * sigma)
            else:
                shift = 0.5 if phase == 0.5 else 0.0
                val = 1.0
                for d in (abs(i + shift - centre) / factor, abs(j + shift - centre) / factor):
                    if d != 0:
                        val *= support * math.sin(math.pi * d) * math.sin(math.pi * d / support) / (math.pi * math.pi * d * d)
                k[i - 1, j - 1] = val
    return k / k.sum()


def down_pad(K, factor):
    """Replication pad of preserve_size=True (models/downsampler.py:54-59)."""
    return int((K - 1) / 2.0) if K % 2 == 1 else int((K - factor) / 2.0)


def downsample(x, kernel, factor, pad):
    """Downsampler.forward (models/downsampler.py:64-71): ReplicationPad2d(pad) + a dense Conv2d(C, C, K, stride=factor)
    whose weight carries `kernel` on the plane diagonal and zeros elsewhere, zero bias."""
    C = x.shape[1]
    k = torch.as_tensor(kernel).to(x.dtype)
    w = torch.zeros(C, C, k.shape[0], k.shape[1], dtype=x.dtype)
    for c in range(C):
        w[c, c] = k
    if pad > 0:
        x = F.pad(x, (pad,) * 4, mode="replicate")
    return F.conv2d(x, w, torch.zeros(C, dtype=x.dtype), stride=factor)


def run(cfg, params, z0, target, noises, sigma, lr, mask=None, record=None, down=None):
    """`len(noises)` iterations of the lean closure: z = z0 + noise*sigma; out = net(z); loss; backward; Adam.
    Returns (losses, last_out).  record(i, out, loss, grads) is called before the Adam step.
    down = (kernel, factor, pad): super-resolution closure, loss = mse(downsample(out), target) (super-resolution.ipynb c10)."""
    opt = Adam(params, lr)
    losses, out = [], None
    for i, nz in enumerate(noises):
        z = z0 + nz * sigma if nz is not None else z0
        out = skip_forward(params, z, cfg)
        loss = mse_loss(out if down is None else downsample(out, *down), target, mask)
        grads = torch.autograd.grad(loss, params)
        if record is not None:
            record(i, out.detach(), loss.item(), grads)
        losses.append(loss.item())
        opt.step(grads)
    return losses, out.detach()


def psnr(a, b):
    """skimage.measure.compare_psnr for float images in [0,1] (data_range 1)."""
    mse = float(np.mean((np.asarray(a, dtype=np.float64) - np.asarray(b, dtype=np.float64)) ** 2))
    return 10.0 * math.log10(1.0 / mse)
