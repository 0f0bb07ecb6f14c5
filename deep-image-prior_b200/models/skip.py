"""models.skip(): the hourglass "skip" network builder with the reference's signature (reference: models/skip.py:5-100).

The returned object is an nn.Sequential whose children, parameter names, parameter order and initialisation RNG order
are those of the reference (so state_dict()s are interchangeable and torch.manual_seed(s) gives identical weights), but
calling it does NOT interpret the module tree: for the configurations of BASELINE.json the whole forward + backward runs
in the hand-written sm_90a engine (libdip.so) through one autograd node.  There is no silent fallback: unsupported
configurations or CPU tensors raise unless the caller opts in to stock-torch execution with
`models.allow_torch_execution(True)` (used by the CPU tests that compare the tree with the reference's).
"""
import torch
import torch.nn as nn

from .common import Concat, act, bn, conv

_ALLOW_TORCH = False


def allow_torch_execution(flag=True):
    """Opt in/out of executing un-accelerated configurations with stock torch modules (default: off)."""
    global _ALLOW_TORCH
    _ALLOW_TORCH = bool(flag)


def _numbered(*mods):
    s = nn.Sequential()
    for m in mods:
        s.add(m)
    return s


def _as_list(v, n):
    return list(v) if isinstance(v, (list, tuple)) else [v] * n


class _EngineFn(torch.autograd.Function):
    """One autograd node for the whole network: forward = dip_forward, backward = dip_backward."""

    @staticmethod
    def forward(ctx, net, z, anchor):
        ctx.net = net
        ctx.want_dz = bool(ctx.needs_input_grad[1])
        out = net._engine_forward(z, want_dz=ctx.want_dz)
        # the saved activations / BatchNorm statistics live in the plan's workspace, one set per plan: remember which
        # forward they belong to (any later forward on the same network overwrites them)
        ctx.plan = net._dip_active_plan
        ctx.generation = net._dip_generation
        return out

    @staticmethod
    def backward(ctx, dout):
        net = ctx.net
        if net._dip_generation != ctx.generation or net._dip_active_plan is not ctx.plan:
            raise RuntimeError(
                "dip-b200: backward() of a forward pass whose saved activations were overwritten by a later forward of "
                "the same network (the engine keeps ONE set of activations per network: call backward() before the next "
                "net(...) -- torch.no_grad() previews included -- or use a second network object)")
        net._engine_backward(dout)
        # OPT_OVER = 'net,input' (utils/common_utils.py:47-49): the input is a leaf that is optimised too
        dz = ctx.plan.input_grad() if ctx.want_dz else None
        return None, dz, None


class SkipNet(nn.Sequential):
    """nn.Sequential with the reference's layout whose __call__ runs on the dip-b200 engine."""

    def __init__(self):
        super().__init__()
        self._dip_spec = None        # dict of engine arguments, or None if the configuration is not accelerated
        self._dip_why = None         # reason when _dip_spec is None
        self._dip_plans = {}
        self._dip_grad_arena = None
        self._dip_anchor = None
        self._dip_generation = 0     # bumped by every engine forward (guards backward against stale activations)
        self._dip_active_plan = None
        # 'tf32' (wgmma tf32, default) | 'fp32' (exact CUDA-core parity mode) | 'bf16' (wgmma on bf16
        # operands, fp32 accumulate / master weights / BatchNorm / Adam: BASELINE.json configs[2])
        self.precision = 'tf32'

    # ---- engine plumbing -------------------------------------------------------------------------------------
    def _apply(self, fn, *args, **kwargs):
        # .type() / .cuda() / .to() / .float() replace parameter and buffer storage: rebuild the engine binding
        self._dip_cache = None
        return super()._apply(fn, *args, **kwargs)

    def _engine_state(self, z, want_dz=False):
        """(plan, parameters) for input z; everything derived from the module tree is cached between calls and
        re-validated cheaply (storage of the first / last parameter and of one BatchNorm buffer): after the per-step
        loss read-back of a notebook closure the GPU idles until this returns, so it must cost microseconds."""
        import dip_engine as de
        try:
            prec = {'tf32': de.PRECISION_TF32, 'fp32': de.PRECISION_FP32, 'bf16': de.PRECISION_BF16}[self.precision]
        except KeyError:
            raise ValueError("dip-b200: net.precision must be 'tf32', 'fp32' or 'bf16', not %r" % (self.precision,))
        key = (int(z.shape[2]), int(z.shape[3]), z.device, prec, bool(want_dz))
        c = getattr(self, '_dip_cache', None)
        if c is not None and c['key'] == key:
            ps = c['params']
            if (ps[0].data_ptr() == c['p0'] and ps[-1].data_ptr() == c['p1'] and c['bn0'].data_ptr() == c['b0']
                    and ps[0].dtype == torch.float32):
                return c['plan'], ps
        return self._engine_state_slow(z, key, prec)

    def _engine_state_slow(self, z, key, prec):
        import dip_engine as de
        spec = self._dip_spec
        H, W = key[0], key[1]
        pkey = (H, W, str(z.device), prec, key[4], spec.get('pad', 'reflection'), spec.get('act_fun', 'LeakyReLU'))
        plan = self._dip_plans.get(pkey)
        if plan is None:
            plan = de.Plan(spec['in_channels'], spec['out_channels'], spec['num_scales'], spec['channels'],
                           spec['skip_channels'], spec['bilinear'], H, W, precision=prec, device=z.device,
                           need_sigmoid=spec['need_sigmoid'], input_grad=key[4], channels_up=spec.get('channels_up'),
                           downsample_mode=spec.get('downsample_mode', 'stride'), pad=spec.get('pad', 'reflection'),
                           act=spec.get('act_fun', 'LeakyReLU'))
            self._dip_plans[pkey] = plan
        params = list(self.parameters())
        for p in params:
            if p.device != z.device or p.dtype != torch.float32:
                raise RuntimeError("dip-b200: parameters must be float32 on the input's device "
                                   "(use net.type(torch.cuda.FloatTensor))")
        total = sum(p.numel() for p in params)
        arena = self._dip_grad_arena
        if arena is None or arena.device != z.device or arena.numel() != total:
            arena = torch.zeros(total, dtype=torch.float32, device=z.device)
            self._dip_grad_arena = arena
            views, o = [], 0
            for p in params:
                views.append(arena[o:o + p.numel()].view_as(p))
                o += p.numel()
            self._dip_grad_views = views
        running = []
        for m in self.modules():
            if isinstance(m, nn.BatchNorm2d):
                running += [m.running_mean, m.running_var, m.num_batches_tracked]
        plan.bind([p.data for p in params], self._dip_grad_views, running)
        self._dip_cache = dict(key=key, plan=plan, params=params, p0=params[0].data_ptr(), p1=params[-1].data_ptr(),
                               bn0=running[0], b0=running[0].data_ptr())
        return plan, params

    def _engine_forward(self, z, want_dz=False):
        plan, _ = self._engine_state(z, want_dz)
        self._dip_active_plan = plan
        self._dip_generation += 1
        zc = z.detach().contiguous()
        return plan.forward(zc)

    def _engine_backward(self, dout):
        plan = self._dip_active_plan
        c = getattr(self, '_dip_cache', None)
        params = c['params'] if c is not None else list(self.parameters())
        views = self._dip_grad_views
        # gradients already attached to the arena (no zero_grad() since the last backward) must be accumulated
        stale = [p.grad is not None and p.grad.data_ptr() == v.data_ptr() for p, v in zip(params, views)]
        prev = self._dip_grad_arena.clone() if any(stale) else None
        plan.backward(dout.contiguous())
        if prev is not None:
            self._dip_grad_arena.add_(prev)
        for p, v, s in zip(params, views, stale):
            if not p.requires_grad:
                continue
            if p.grad is None:
                p.grad = v
            elif not s:
                p.grad.add_(v)

    # ---- nn.Module surface -----------------------------------------------------------------------------------
    def forward(self, x):
        if self._dip_spec is not None and x.is_cuda:
            if x.dim() != 4 or x.shape[0] != 1 or x.shape[1] != self._dip_spec['in_channels']:
                raise ValueError("dip-b200: expected input of shape 1 x %d x H x W" % self._dip_spec['in_channels'])
            if x.dtype != torch.float32:
                # torch would raise a dtype mismatch against the float32 weights (e.g. get_noise(..., 'meshgrid')
                # without .type(dtype) is float64); the engine reads raw fp32 storage, so it must refuse as well
                raise RuntimeError("dip-b200: expected a float32 input, got %s (use .type(torch.cuda.FloatTensor))" % x.dtype)
            if not self.training:
                # nothing in the reference ever calls .eval() (SURVEY.md 3.5); the engine only implements the
                # training-mode BatchNorm (batch statistics + running-stat update)
                raise NotImplementedError("dip-b200: the engine runs BatchNorm in training mode only (net.eval() is not "
                                          "supported; models.allow_torch_execution(True) + CPU tensors runs stock torch)")
            if not torch.is_grad_enabled():
                return self._engine_forward(x)
            if self._dip_anchor is None or self._dip_anchor.device != x.device:
                self._dip_anchor = torch.zeros(1, device=x.device, requires_grad=True)
            return _EngineFn.apply(self, x, self._dip_anchor)
        if _ALLOW_TORCH:
            return super().forward(x)
        if self._dip_spec is None:
            raise NotImplementedError("dip-b200: this skip() configuration is not accelerated by the engine (%s). "
                                      "Call models.allow_torch_execution(True) to run it with stock torch modules."
                                      % self._dip_why)
        raise RuntimeError("dip-b200: the accelerated path needs CUDA tensors (net.type(torch.cuda.FloatTensor)); "
                           "there is no CPU fallback. models.allow_torch_execution(True) opts in to stock torch.")


def skip(num_input_channels=2, num_output_channels=3,
         num_channels_down=[16, 32, 64, 128, 128], num_channels_up=[16, 32, 64, 128, 128],
         num_channels_skip=[4, 4, 4, 4, 4],
         filter_size_down=3, filter_size_up=3, filter_skip_size=1,
         need_sigmoid=True, need_bias=True,
         pad='zero', upsample_mode='nearest', downsample_mode='stride', act_fun='LeakyReLU',
         need1x1_up=True):
    """Assembles the encoder-decoder with skip connections (same arguments as the reference's models.skip)."""
    assert len(num_channels_down) == len(num_channels_up) == len(num_channels_skip)
    n = len(num_channels_down)
    upsample_mode = _as_list(upsample_mode, n)
    downsample_mode = _as_list(downsample_mode, n)
    filter_size_down = _as_list(filter_size_down, n)
    filter_size_up = _as_list(filter_size_up, n)

    # 1) leaves, created in the reference's construction order (= RNG draw order): per scale skip-conv, down convs,
    #    up conv, 1x1 conv; the RGB head last (reference: models/skip.py:45-98).
    leaves = []
    depth = num_input_channels
    for i in range(n):
        k_deeper = num_channels_up[i + 1] if i < n - 1 else num_channels_down[i]
        lv = {}
        lv['cat_bn'] = bn(num_channels_skip[i] + k_deeper)
        if num_channels_skip[i] != 0:
            lv['skip'] = (conv(depth, num_channels_skip[i], filter_skip_size, bias=need_bias, pad=pad),
                          bn(num_channels_skip[i]), act(act_fun))
        lv['down1'] = (conv(depth, num_channels_down[i], filter_size_down[i], 2, bias=need_bias, pad=pad,
                            downsample_mode=downsample_mode[i]), bn(num_channels_down[i]), act(act_fun))
        lv['down2'] = (conv(num_channels_down[i], num_channels_down[i], filter_size_down[i], bias=need_bias, pad=pad),
                       bn(num_channels_down[i]), act(act_fun))
        lv['upsample'] = nn.Upsample(scale_factor=2, mode=upsample_mode[i])
        lv['up'] = (conv(num_channels_skip[i] + k_deeper, num_channels_up[i], filter_size_up[i], 1, bias=need_bias,
                         pad=pad), bn(num_channels_up[i]), act(act_fun))
        if need1x1_up:
            lv['up1x1'] = (conv(num_channels_up[i], num_channels_up[i], 1, bias=need_bias, pad=pad),
                           bn(num_channels_up[i]), act(act_fun))
        leaves.append(lv)
        depth = num_channels_down[i]
    head = conv(num_channels_up[0], num_output_channels, 1, bias=need_bias, pad=pad)

    # 2) tree, assembled bottom-up with the reference's child numbering
    def level_modules(i):
        lv = leaves[i]
        deeper_mods = list(lv['down1']) + list(lv['down2'])
        if i < n - 1:
            deeper_mods.append(_numbered(*level_modules(i + 1)))
        deeper_mods.append(lv['upsample'])
        deeper = _numbered(*deeper_mods)
        first = Concat(1, _numbered(*lv['skip']), deeper) if 'skip' in lv else deeper
        mods = [first, lv['cat_bn']] + list(lv['up'])
        if need1x1_up:
            mods += list(lv['up1x1'])
        return mods

    net = SkipNet()
    for m in level_modules(0):
        net.add(m)
    net.add(head)
    if need_sigmoid:
        net.add(nn.Sigmoid())

    # 3) is this one of the configurations the engine executes?
    why = None
    chans = set(num_channels_down) | set(num_channels_up)
    if any(c % 8 != 0 or not 8 <= c <= 128 for c in chans):
        why = 'num_channels_down/up must be multiples of 8 in [8, 128]'
    elif not (set(num_channels_skip) <= {0, 4} or (set(num_channels_skip) == {128} and chans == {128})):
        why = 'num_channels_skip must be 0 or 4 per scale (or 128 at every scale of a 128-wide network)'
    elif set(filter_size_down) != {3} or set(filter_size_up) != {3} or filter_skip_size != 1:
        why = 'filter sizes must be 3/3/1'
    elif set(downsample_mode) not in ({'stride'}, {'avg'}):
        why = "downsample_mode must be 'stride' or 'avg' (at every scale)"
    elif not (isinstance(act_fun, str) and act_fun in ('LeakyReLU', 'Swish', 'ELU', 'none')):
        why = "act_fun must be 'LeakyReLU', 'Swish', 'ELU' or 'none' (a module class is not accelerated)"
    elif not (need_bias and need1x1_up):
        why = 'need_bias and need1x1_up must be True'
    elif any(m not in ('bilinear', 'nearest') for m in upsample_mode):
        why = "upsample_mode must be 'bilinear' or 'nearest' (per scale)"
    elif not (1 <= num_output_channels <= 4 and 1 <= num_input_channels <= 128):
        why = 'num_output_channels in 1..4 and num_input_channels in 1..128'
    if why is None:
        uniform = chans == {128} and len(set(num_channels_skip)) == 1
        net._dip_spec = dict(in_channels=num_input_channels, out_channels=num_output_channels, num_scales=n,
                             channels=128 if uniform else list(num_channels_down),
                             channels_up=None if uniform else list(num_channels_up),
                             skip_channels=num_channels_skip[0] if uniform else list(num_channels_skip),
                             need_sigmoid=bool(need_sigmoid), downsample_mode=downsample_mode[0],
                             # models/common.py:conv: only pad == 'reflection' inserts ReflectionPad2d, any other value
                             # is Conv2d(padding=(k-1)//2), i.e. zero padding
                             pad='reflection' if pad == 'reflection' else 'zero',
                             act_fun=act_fun,
                             bilinear=(upsample_mode[0] == 'bilinear' if len(set(upsample_mode)) == 1
                                       else [m == 'bilinear' for m in upsample_mode]))
    else:
        net._dip_why = why
    return net
