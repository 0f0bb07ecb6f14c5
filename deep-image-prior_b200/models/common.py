"""Building blocks with the reference's names and module-tree numbering (reference: models/common.py).

The blocks are ordinary torch modules because they double as the parameter holders / state_dict layout of the
network; on the accelerated path their forward() is never called -- SkipNet (models/skip.py) hands the whole graph to
the sm_90a engine instead.
"""
import numpy as np
import torch
import torch.nn as nn

from .downsampler import Downsampler


def _append_numbered(self, module):
    # children are numbered from "1" (reference: models/common.py:6-9) -> state_dict keys such as "1.0.1.1.weight"
    self.add_module(str(len(self) + 1), module)


torch.nn.Module.add = _append_numbered


class Concat(nn.Module):
    """Runs every branch on the same input, centre-crops to the smallest H x W, concatenates along `dim`
    (reference: models/common.py:11-42)."""

    def __init__(self, dim, *branches):
        super().__init__()
        self.dim = dim
        for i, b in enumerate(branches):
            self.add_module(str(i), b)

    def forward(self, x):
        ys = [b(x) for b in self._modules.values()]
        h = min(y.shape[2] for y in ys)
        w = min(y.shape[3] for y in ys)
        cropped = []
        for y in ys:
            if y.shape[2] != h or y.shape[3] != w:
                t, l = (y.shape[2] - h) // 2, (y.shape[3] - w) // 2
                y = y[:, :, t:t + h, l:l + w]
            cropped.append(y)
        return torch.cat(cropped, dim=self.dim)

    def __len__(self):
        return len(self._modules)


class GenNoise(nn.Module):
    """Fresh N(0,1) tensor shaped like the input but with `dim2` channels (reference: models/common.py:45-60)."""

    def __init__(self, dim2):
        super().__init__()
        self.dim2 = dim2

    def forward(self, x):
        shape = list(x.size())
        shape[1] = self.dim2
        return torch.zeros(shape, dtype=x.dtype, device=x.device).normal_()


class Swish(nn.Module):
    """x * sigmoid(x) (reference: models/common.py:63-73)."""

    def __init__(self):
        super().__init__()
        self.s = nn.Sigmoid()

    def forward(self, x):
        return x * self.s(x)


def act(act_fun='LeakyReLU'):
    """Activation by name or by module class (reference: models/common.py:76-92)."""
    if not isinstance(act_fun, str):
        return act_fun()
    table = {'LeakyReLU': lambda: nn.LeakyReLU(0.2, inplace=True), 'Swish': Swish, 'ELU': nn.ELU,
             'none': nn.Sequential}
    assert act_fun in table, 'unknown activation ' + act_fun
    return table[act_fun]()


def bn(num_features):
    return nn.BatchNorm2d(num_features)


def conv(in_f, out_f, kernel_size, stride=1, bias=True, pad='zero', downsample_mode='stride'):
    """[ReflectionPad2d] + Conv2d + [AvgPool/MaxPool/Lanczos downsampler] (reference: models/common.py:99-124)."""
    down = None
    if stride != 1 and downsample_mode != 'stride':
        if downsample_mode == 'avg':
            down = nn.AvgPool2d(stride, stride)
        elif downsample_mode == 'max':
            down = nn.MaxPool2d(stride, stride)
        elif downsample_mode in ('lanczos2', 'lanczos3'):
            down = Downsampler(n_planes=out_f, factor=stride, kernel_type=downsample_mode, phase=0.5,
                               preserve_size=True)
        else:
            assert False, 'unknown downsample_mode ' + str(downsample_mode)
        stride = 1
    p = int((kernel_size - 1) / 2)
    mods = []
    if pad == 'reflection':
        mods.append(nn.ReflectionPad2d(p))
        p = 0
    mods.append(nn.Conv2d(in_f, out_f, kernel_size, stride, padding=p, bias=bias))
    if down is not None:
        mods.append(down)
    return nn.Sequential(*mods)
