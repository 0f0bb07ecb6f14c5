"""The CPU oracle (oracle/dip_oracle.py) and the fp64 stage references (tests/stage_ref.py) for networks built with zero
padding (test infrastructure).

models.skip's `pad` (reference: models/common.py:114-120): only 'reflection' puts nn.ReflectionPad2d(k // 2) in front of
a conv; every other value gives Conv2d(padding=k // 2), i.e. zero padding.  Both references pad by reflection, and both
reach the padding through module-level functions looked up at call time: the oracle's `_conv`, and stage_ref's
`reflect_pad` (every padded conv input) and `fold` (its adjoint, on every padded gradient).  `padding(cfg)` swaps in the
zero-padding forms of exactly those functions while it is active, when `cfg.pad` is not 'reflection' (the default when a
SkipConfig carries no `pad`); everything else (bf16 operand rounding, layouts, tolerances) is the references' own code.
"""
import contextlib

import torch.nn.functional as F

from oracle import dip_oracle as O
import stage_ref as SR


def pad_of(cfg):
    return getattr(cfg, "pad", "reflection")


def _conv_zero_pad(x, w, b, stride=1):
    k = w.shape[-1]
    if k > 1:
        x = F.pad(x, (k // 2,) * 4)   # nn.Conv2d(padding=k // 2)
    if O._OPERAND_ROUND == "bf16" and w.shape[0] >= O._MIN_TENSOR_CORE_WIDTH:
        return O._ConvBf16Operands.apply(x, w, b, stride)
    return F.conv2d(x, w, b, stride=stride)


def zero_pad(x):
    """Conv2d(padding=1) in the engine's layout: [H][W][C] -> [(H+2)][(W+2)][C] with a zero halo"""
    return SR.hwc(F.pad(SR.nchw(x), (1, 1, 1, 1)))


def zero_fold(gp):
    """adjoint of zero_pad: the interior of the padded gradient (the halo's gradient is dropped)"""
    return gp[1:-1, 1:-1]


@contextlib.contextmanager
def padding(cfg):
    if pad_of(cfg) == "reflection":
        yield
        return
    saved = O._conv, SR.reflect_pad, SR.fold
    O._conv, SR.reflect_pad, SR.fold = _conv_zero_pad, zero_pad, zero_fold
    try:
        yield
    finally:
        O._conv, SR.reflect_pad, SR.fold = saved


# ---- oracle
def skip_forward(params, z, cfg, tape=None):
    with padding(cfg):
        return O.skip_forward(params, z, cfg, tape)


def run(cfg, params, z0, target, noises, sigma, lr, **kw):
    with padding(cfg):
        return O.run(cfg, params, z0, target, noises, sigma, lr, **kw)


# ---- stage references (same arguments as stage_ref.forward / stage_ref.backward)
def stage_forward(cfg, params, src, mode, refs, **kw):
    with padding(cfg):
        return SR.forward(cfg, params, src, mode, refs, **kw)


def stage_backward(cfg, params, src, mode, refs, dout, **kw):
    with padding(cfg):
        return SR.backward(cfg, params, src, mode, refs, dout, **kw)
