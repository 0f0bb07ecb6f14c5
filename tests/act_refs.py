"""The CPU oracle (oracle/dip_oracle.py) and the fp64 stage references (tests/stage_ref.py) for networks built with
act_fun 'Swish', 'ELU' or 'none' (test infrastructure).

models.skip's act_fun (reference: models/common.py:76-92) is the activation behind every BatchNorm except the concat's:
'LeakyReLU' = nn.LeakyReLU(0.2), 'Swish' = x * sigmoid(x), 'ELU' = nn.ELU() (alpha = 1), 'none' = nn.Sequential().  Both
references apply LeakyReLU, and both reach it through module-level names looked up at call time: the oracle's `_act`, and
stage_ref's `Bn` (whose out() / backward() apply the activation and its derivative).  `activation(cfg)` swaps in the
forms for cfg.act_fun (absent: 'LeakyReLU', which swaps nothing) while it is active.  CatBn keeps its own base class and
is only ever used with act=False, so the concat BatchNorm is unaffected.

None of the three has a jump in its first derivative (the LeakyReLU boundary band of stage_ref exists because that
derivative jumps at 0), so the elementwise backward checks exclude no element and the reductions get no flip term.  The
tolerances are stage_ref's own plus one term that LeakyReLU never needs, because its derivative is exact off the band:
the kernels evaluate f'(y) in fp32, at the fp32 pre-activation fma(x, scale, shift).  That error enters dz = g f'(y)
like a gradient computed on the fly (stage_ref.Bn.backward's `gtol`, propagated the same way):
  |g| (F2 dy + 8 2^-23 (1 + |y|)),  dy = 2 2^-23 (|x scale| + |shift| + |mean scale|),  F2 = sup |f''| (Swish 0.5, ELU 1)
(dy bounds the rounding of the fp32 pre-activation, the second term that of the fp32 evaluation of f').  It matters where the BatchNorm backward cancels: at the deepest level of a 64 x 96 'avg' network a channel has 6 pixels,
and dx = scale (dz - mean(dz) - xhat mean(dz xhat)) keeps only a small part of dz.  'none' has f' = 1 exactly.
"""
import contextlib

import torch
import torch.nn.functional as F

from oracle import dip_oracle as O
import pad_refs as PR
import stage_ref as SR

KINDS = ("LeakyReLU", "Swish", "ELU", "none")
_BN = SR.Bn   # stage_ref's own (LeakyReLU) class, the base of the swapped-in ones


def act_of(cfg):
    return getattr(cfg, "act_fun", "LeakyReLU")


def _swish(y):
    return y * torch.sigmoid(y)


def _swish_grad(y):
    s = torch.sigmoid(y)
    return s * (1 + y * (1 - s))


FWD = {"Swish": _swish, "ELU": F.elu, "none": lambda y: y}
GRAD = {"Swish": _swish_grad, "ELU": lambda y: torch.where(y > 0, torch.ones_like(y), torch.exp(y)),
        "none": torch.ones_like}
F2 = {"Swish": 0.5, "ELU": 1.0, "none": 0.0}   # sup |f''|


def bn_class(kind):
    """stage_ref.Bn with activation `kind` (and its derivative) in place of LeakyReLU"""
    f, df = FWD[kind], GRAD[kind]

    class ActBn(_BN):
        def __init__(self, raw, g, b):
            super().__init__(raw, g, b)
            x = raw.double().reshape(-1, raw.shape[-1])
            mean = x.mean(0)
            shift = b.double() - mean * self.scale
            # fp32 derivative error per unit of incoming gradient (module docstring)
            dy = 2 * SR.U23 * ((x * self.scale).abs() + shift.abs() + (mean * self.scale).abs())
            self.dact = 0.0 if kind == "none" else F2[kind] * dy + 8 * SR.U23 * (1 + self.y.abs())

        def out(self, act=True):
            return (f(self.y) if act else self.y).reshape(self.shape)

        def backward(self, gout, act=True, gtol=None):
            go = gout.double().reshape(-1, self.shape[-1])
            xh = self.xhat
            d = df(self.y) if act else torch.ones_like(go)
            dz = go * d
            gt = torch.zeros_like(go) if gtol is None else gtol.double().reshape(-1, self.shape[-1]) * d.abs()
            if act:
                gt = gt + go.abs() * self.dact
            m1, m2 = dz.mean(0), (dz * xh).mean(0)
            dx = self.scale * (dz - m1 - xh * m2)
            f1, f2 = gt.sum(0), (gt * xh.abs()).sum(0)
            tol_dx = SR.mem_tol(dx) + self.scale.abs() * (gt + (f1 + xh.abs() * f2) / self.n)
            excl = torch.zeros_like(go, dtype=torch.bool)
            return dict(dx=dx.reshape(self.shape), tol_dx=tol_dx.reshape(self.shape), excl=excl.reshape(self.shape),
                        dbeta=dz.sum(0), tol_dbeta=SR.RED_REL * dz.abs().sum(0) + f1,
                        dgamma=(dz * xh).sum(0), tol_dgamma=SR.RED_REL * (dz * xh).abs().sum(0) + f2,
                        excl_frac=0.0)

    ActBn.__name__ = ActBn.__qualname__ = "Bn_" + kind
    return ActBn


@contextlib.contextmanager
def activation(cfg):
    kind = act_of(cfg)
    if kind == "LeakyReLU":
        yield
        return
    saved = O._act, SR.Bn
    O._act, SR.Bn = FWD[kind], bn_class(kind)
    try:
        yield
    finally:
        O._act, SR.Bn = saved


@contextlib.contextmanager
def both(cfg):
    """cfg's padding (pad_refs.padding) and activation"""
    with PR.padding(cfg), activation(cfg):
        yield


# ---- oracle
def skip_forward(params, z, cfg, tape=None):
    with both(cfg):
        return O.skip_forward(params, z, cfg, tape)


def run(cfg, params, z0, target, noises, sigma, lr, **kw):
    with both(cfg):
        return O.run(cfg, params, z0, target, noises, sigma, lr, **kw)


# ---- stage references (same arguments as stage_ref.forward / stage_ref.backward)
def stage_forward(cfg, params, src, mode, refs, **kw):
    with both(cfg):
        return SR.forward(cfg, params, src, mode, refs, **kw)


def stage_backward(cfg, params, src, mode, refs, dout, **kw):
    with both(cfg):
        return SR.backward(cfg, params, src, mode, refs, dout, **kw)
