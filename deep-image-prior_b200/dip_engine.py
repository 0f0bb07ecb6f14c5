"""ctypes binding of libdip.so (C ABI declared in include/dip.h).

This is the only place where Python touches the native engine.  PyTorch is used for device memory, streams and
autograd plumbing; every FLOP of the hot path runs in the hand-written sm_90a kernels of libdip.so.
The library is mandatory: there is no CPU or eager-PyTorch fallback for the accelerated path.
"""
import ctypes
import os
import subprocess

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("DIP_LIB") or os.path.join(_HERE, "libdip.so")  # DIP_LIB: experiment builds

PRECISION_TF32 = 0
PRECISION_FP32 = 1
PRECISION_BF16 = 2

PAD_REFLECTION = 0   # dip_plan_opts.pad_mode: nn.ReflectionPad2d(1) before every 3x3 conv (models.skip pad='reflection')
PAD_ZERO = 1         # Conv2d(padding=1): every other value of models.skip's `pad` (reference: models/common.py:114-120)

# dip_plan_opts.act_fun: models.skip's act_fun string (reference: models/common.py:76-92), the activation behind every
# BatchNorm except the concat's
ACT_LEAKY_RELU = 0   # 'LeakyReLU': nn.LeakyReLU(0.2)
ACT_SWISH = 1        # 'Swish': x * sigmoid(x)
ACT_ELU = 2          # 'ELU': nn.ELU() (alpha = 1)
ACT_NONE = 3         # 'none': nn.Sequential(), the identity
ACT_FUNS = {"LeakyReLU": ACT_LEAKY_RELU, "Swish": ACT_SWISH, "ELU": ACT_ELU, "none": ACT_NONE}


class NetDesc(ctypes.Structure):
    _fields_ = [
        ("in_channels", ctypes.c_int),
        ("out_channels", ctypes.c_int),
        ("num_scales", ctypes.c_int),
        ("channels", ctypes.c_int),
        ("skip_channels", ctypes.c_int),
        ("upsample_bilinear", ctypes.c_int),
        ("need_sigmoid", ctypes.c_int),
        ("precision", ctypes.c_int),
        ("upsample_mask", ctypes.c_int),
        ("input_grad", ctypes.c_int),
        ("channels_down", ctypes.c_int * 8),
        ("channels_up", ctypes.c_int * 8),
        ("channels_skip", ctypes.c_int * 8),
        ("downsample_mode", ctypes.c_int),
    ]


class Track(ctypes.Structure):
    """dip_track (include/dip.h): the denoising closure's EMA, PSNRs and back-tracking inside the runner"""
    _fields_ = [("gt", ctypes.c_void_p), ("out_avg", ctypes.c_void_p), ("snapshot", ctypes.c_void_p),
                ("state", ctypes.c_void_p), ("records", ctypes.c_void_p), ("exp_weight", ctypes.c_double),
                ("show_every", ctypes.c_int), ("backtrack_db", ctypes.c_double)]


RECORD = 6                     # doubles per tracked iteration: loss, psnr_target, psnr_gt, psnr_gt_sm, i, action
ACTION_NONE, ACTION_SAVED, ACTION_RESTORED = 0, 1, 2


class PlanOpts(ctypes.Structure):
    """dip_plan_opts (include/dip.h): PlanOpts(pad_mode, act_fun); a field left out is 0 (reflection, LeakyReLU)"""
    _fields_ = [("pad_mode", ctypes.c_int), ("act_fun", ctypes.c_int)]


_lib = None

# every symbol include/dip.h declares (checked by tests/test_abi.py)
ABI_SYMBOLS = [
    "dip_last_error", "dip_version", "dip_plan_workspace_bytes", "dip_plan_create", "dip_plan_destroy",
    "dip_plan_num_params", "dip_plan_num_bn", "dip_plan_param_numel", "dip_plan_bind", "dip_forward", "dip_backward",
    "dip_loss_mse", "dip_noise_perturb", "dip_adam_create", "dip_adam_destroy", "dip_adam_bind", "dip_adam_step",
    "dip_run_iterations", "dip_plan_buffer", "dip_plan_num_launches", "dip_plan_set_timing", "dip_plan_get_timing", "dip_plan_get_timing_records", "dip_op_scratch_bytes", "dip_op_conv_fprop",
    "dip_op_conv_dgrad", "dip_op_conv_wgrad", "dip_op_conv_dgrad_s2",
    "dip_lanczos_down_out_size", "dip_lanczos_down_fwd", "dip_lanczos_down_bwd", "dip_plan_set_downsampler",
    "dip_input_grad", "dip_plan_workspace_bytes_opts", "dip_plan_create_opts",
    "dip_track_state_bytes", "dip_run_iterations_tracked",
]


def build(verbose=False):
    """Compile libdip.so in-tree with nvcc for sm_90a (no GPU needed)."""
    out = subprocess.run([os.path.join(_HERE, "build.sh")], capture_output=True, text=True)
    if verbose or out.returncode != 0:
        print(out.stdout)
        print(out.stderr)
    if out.returncode != 0:
        raise RuntimeError("building libdip.so failed")
    return LIB_PATH


def lib():
    """Load libdip.so; raises loudly if it is missing (no fallback path exists)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "libdip.so not found at %s -- run deep-image-prior_b200/build.sh (or __graft_entry__.build()). "
            "The dip-b200 hot path has no CPU/eager fallback." % LIB_PATH)
    L = ctypes.CDLL(LIB_PATH)
    vp, i32, i64, u64, f32, f64, sz = (ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_uint64,
                                       ctypes.c_float, ctypes.c_double, ctypes.c_size_t)
    pvp = ctypes.POINTER(ctypes.c_void_p)
    L.dip_last_error.restype = ctypes.c_char_p
    L.dip_version.restype = i32
    L.dip_plan_workspace_bytes.restype = sz
    L.dip_plan_workspace_bytes.argtypes = [ctypes.POINTER(NetDesc), i32, i32]
    L.dip_plan_create.argtypes = [ctypes.POINTER(NetDesc), i32, i32, vp, sz, pvp]
    L.dip_plan_workspace_bytes_opts.restype = sz
    L.dip_plan_workspace_bytes_opts.argtypes = [ctypes.POINTER(NetDesc), i32, i32, ctypes.POINTER(PlanOpts)]
    L.dip_plan_create_opts.argtypes = [ctypes.POINTER(NetDesc), i32, i32, ctypes.POINTER(PlanOpts), vp, sz, pvp]
    L.dip_plan_destroy.argtypes = [vp]
    L.dip_plan_destroy.restype = None
    L.dip_plan_num_params.argtypes = [vp]
    L.dip_plan_num_bn.argtypes = [vp]
    L.dip_plan_param_numel.argtypes = [vp, i32]
    L.dip_plan_param_numel.restype = i64
    L.dip_plan_bind.argtypes = [vp, pvp, pvp, pvp, i32]
    L.dip_forward.argtypes = [vp, vp, vp, f32, vp, vp]
    L.dip_backward.argtypes = [vp, vp, vp]
    L.dip_loss_mse.argtypes = [vp, vp, vp, i32, i32, vp, vp, vp]
    L.dip_noise_perturb.argtypes = [vp, vp, f32, u64, u64, sz, vp]
    L.dip_adam_create.argtypes = [i32, ctypes.POINTER(i64), pvp]
    L.dip_adam_destroy.argtypes = [vp]
    L.dip_adam_destroy.restype = None
    L.dip_adam_bind.argtypes = [vp, pvp, pvp, pvp, pvp]
    L.dip_adam_step.argtypes = [vp, f64, f64, f64, f64, i32, vp]
    L.dip_run_iterations.argtypes = [vp, vp, vp, vp, vp, f32, u64, i32, i32, f64, vp, vp, vp]
    L.dip_track_state_bytes.restype = sz
    L.dip_run_iterations_tracked.argtypes = [vp, vp, vp, vp, vp, f32, u64, i32, i32, f64, vp, vp, ctypes.POINTER(Track), vp]
    L.dip_plan_buffer.argtypes = [vp, ctypes.c_char_p, pvp, ctypes.POINTER(i32)]
    L.dip_plan_num_launches.argtypes = [vp, ctypes.POINTER(i32), ctypes.POINTER(i32)]
    L.dip_plan_set_timing.argtypes = [vp, i32]
    L.dip_plan_get_timing.argtypes = [vp, ctypes.POINTER(f64), ctypes.POINTER(f64), ctypes.POINTER(i32)]
    L.dip_plan_get_timing_records.argtypes = [vp, i32, ctypes.POINTER(i32), ctypes.POINTER(f64), ctypes.POINTER(f64)]
    L.dip_op_scratch_bytes.restype = sz
    L.dip_op_conv_fprop.argtypes = [vp, i32, i32, i32, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp, i32, i32, vp, i32,
                                    vp, vp]
    L.dip_op_conv_dgrad.argtypes = [vp, i32, i32, vp, i32, i32, i32, i32, vp, i32, i32, i32, vp, vp]
    L.dip_op_conv_dgrad_s2.argtypes = [vp, i32, i32, vp, i32, i32, i32, vp, i32, vp, vp]
    L.dip_op_conv_wgrad.argtypes = [vp, i32, i32, vp, i32, i32, i32, i32, i32, i32, i32, i32, i32, i32, vp, i32, vp, vp]
    L.dip_lanczos_down_out_size.argtypes = [i32, i32, i32, i32]
    L.dip_lanczos_down_fwd.argtypes = [vp, i32, i32, i32, vp, i32, i32, i32, vp, vp]
    L.dip_lanczos_down_bwd.argtypes = [vp, i32, i32, i32, vp, i32, i32, i32, vp, vp]
    L.dip_plan_set_downsampler.argtypes = [vp, ctypes.POINTER(f32), i32, i32, i32]
    L.dip_input_grad.argtypes = [vp, vp, vp]
    _lib = L
    return L


def check(rc):
    if rc != 0:
        raise RuntimeError("libdip: " + lib().dip_last_error().decode())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def _ptr_array(tensors):
    arr = (ctypes.c_void_p * len(tensors))()
    for i, t in enumerate(tensors):
        arr[i] = t.data_ptr()
    return arr


class Plan:
    """A compiled schedule for one skip network at one input size (dip_plan in include/dip.h)."""

    def __init__(self, in_channels, out_channels, num_scales, channels, skip_channels, bilinear, H, W,
                 precision=PRECISION_TF32, device=None, need_sigmoid=True, input_grad=False, channels_up=None,
                 downsample_mode="stride", pad="reflection", act="LeakyReLU"):
        """channels / skip_channels: one width for every scale, or per-scale sequences (num_channels_down / num_channels_skip
        of models.skip; channels_up = num_channels_up, default = channels).  pad: 'reflection' or 'zero' (the padding of
        every 3x3 conv).  act: 'LeakyReLU', 'Swish', 'ELU' or 'none' (models.skip's act_fun)."""
        L = lib()
        if pad not in ("reflection", "zero"):
            raise ValueError("dip-b200: Plan(pad=...) must be 'reflection' or 'zero', not %r" % (pad,))
        if not isinstance(act, str) or act not in ACT_FUNS:
            raise ValueError("dip-b200: Plan(act=...) must be one of %s, not %r" % (", ".join(map(repr, ACT_FUNS)), act))
        self.opts = PlanOpts(PAD_REFLECTION if pad == "reflection" else PAD_ZERO, ACT_FUNS[act])
        self.pad, self.act = pad, act
        per_scale = None
        if isinstance(channels, (list, tuple)) or isinstance(skip_channels, (list, tuple)) or channels_up is not None:
            as_list = lambda x: list(x) if isinstance(x, (list, tuple)) else [x] * num_scales   # noqa: E731
            per_scale = (as_list(channels), as_list(channels if channels_up is None else channels_up), as_list(skip_channels))
            assert all(len(x) == num_scales for x in per_scale) and num_scales <= 8
            channels, skip_channels = 0, 0
        if not torch.cuda.is_available():
            raise RuntimeError("dip-b200 needs a CUDA device (sm_90a); none is visible")
        self.device = torch.device(device if device is not None else "cuda:%d" % torch.cuda.current_device())
        # bilinear: one flag for every scale, or a per-scale sequence (flash-no-flash.ipynb c8)
        if isinstance(bilinear, (list, tuple)):
            assert len(bilinear) == num_scales
            mask = sum(1 << i for i, b in enumerate(bilinear) if b)
            self.desc = NetDesc(in_channels, out_channels, num_scales, channels, skip_channels, -1, int(bool(need_sigmoid)),
                                precision, mask, int(bool(input_grad)))
        else:
            self.desc = NetDesc(in_channels, out_channels, num_scales, channels, skip_channels, int(bool(bilinear)),
                                int(bool(need_sigmoid)), precision, 0, int(bool(input_grad)))
        self.desc.downsample_mode = {"stride": 0, "avg": 1}[downsample_mode]
        if per_scale is not None:
            for name, vals in zip(("channels_down", "channels_up", "channels_skip"), per_scale):
                arr = getattr(self.desc, name)
                for i, x in enumerate(vals):
                    arr[i] = int(x)
        self.H, self.W = H, W
        nbytes = L.dip_plan_workspace_bytes_opts(ctypes.byref(self.desc), H, W, ctypes.byref(self.opts))
        if nbytes == 0:
            raise NotImplementedError("libdip: " + L.dip_last_error().decode())
        with torch.cuda.device(self.device):
            self.workspace = torch.empty(nbytes + 512, dtype=torch.uint8, device=self.device)
            base = (self.workspace.data_ptr() + 255) // 256 * 256
            h = ctypes.c_void_p()
            check(L.dip_plan_create_opts(ctypes.byref(self.desc), H, W, ctypes.byref(self.opts), ctypes.c_void_p(base), nbytes,
                                         ctypes.byref(h)))
        self.h = h
        self.n_params = L.dip_plan_num_params(h)
        self.n_bn = L.dip_plan_num_bn(h)
        self.numel = [L.dip_plan_param_numel(h, i) for i in range(self.n_params)]
        self._bound_key = None
        self._keep = None

    def __del__(self):
        try:
            if getattr(self, "h", None) is not None and _lib is not None:
                _lib.dip_plan_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def bind(self, params, grads, running=None):
        key = (tuple(p.data_ptr() for p in params), tuple(g.data_ptr() for g in grads),
               None if running is None else tuple(r.data_ptr() for r in running))
        if key == self._bound_key:
            return
        assert len(params) == self.n_params and len(grads) == self.n_params
        for p, n in zip(params, self.numel):
            assert p.numel() == n and p.dtype == torch.float32 and p.is_contiguous(), "parameter shape mismatch"
        pa, ga = _ptr_array(params), _ptr_array(grads)
        ra, nbt_float = None, 0
        if running is not None:
            assert len(running) == 3 * self.n_bn
            ra = _ptr_array(running)
            kinds = set(r.dtype for r in running[2::3])
            assert kinds in ({torch.int64}, {torch.float32}), kinds
            nbt_float = int(kinds == {torch.float32})
        with torch.cuda.device(self.device):
            check(lib().dip_plan_bind(self.h, pa, ga, ra, nbt_float))
        self._bound_key = key
        self._keep = (params, grads, running)

    def forward(self, z, noise=None, sigma=0.0, out=None):
        if out is None:
            out = torch.empty((1, self.desc.out_channels, self.H, self.W), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            check(lib().dip_forward(self.h, _ptr(z), _ptr(noise), float(sigma), _ptr(out), _stream()))
        return out

    def backward(self, dout):
        with torch.cuda.device(self.device):
            check(lib().dip_backward(self.h, _ptr(dout), _stream()))

    def input_grad(self):
        """dL/d(net_input) of the last backward (plans created with input_grad=True), 1 x C_in x H x W."""
        dz = torch.empty((1, self.desc.in_channels, self.H, self.W), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            check(lib().dip_input_grad(self.h, _ptr(dz), _stream()))
        return dz

    def set_downsampler(self, kernel, factor, pad):
        """Loss of the runner is taken on downsampler(out) (dip_plan_set_downsampler); kernel: K x K taps or None."""
        if kernel is None:
            check(lib().dip_plan_set_downsampler(self.h, None, 0, 1, 0))
            return
        k = torch.as_tensor(kernel, dtype=torch.float32).contiguous().cpu()
        assert k.dim() == 2 and k.shape[0] == k.shape[1]
        arr = (ctypes.c_float * k.numel())(*k.flatten().tolist())
        with torch.cuda.device(self.device):
            check(lib().dip_plan_set_downsampler(self.h, arr, int(k.shape[0]), int(factor), int(pad)))

    def buffer(self, name):
        """Copy of an internal NHWC buffer as a (rows, cols, channels) tensor (tests / debugging)."""
        p = ctypes.c_void_p()
        dims = (ctypes.c_int * 4)()
        check(lib().dip_plan_buffer(self.h, name.encode(), ctypes.byref(p), dims))
        rows, cols, ld, c = dims[0], dims[1], dims[2], dims[3]
        off = p.value - self.workspace.data_ptr()
        if name.endswith("16"):   # bf16 twin of a conv operand (precision mode bf16)
            flat = self.workspace[off:off + rows * cols * ld * 2].view(torch.bfloat16)
        else:
            flat = self.workspace[off:off + rows * cols * ld * 4].view(torch.float32)
        return flat.view(rows, cols, ld)[:, :, :c].clone()

    def set_timing(self, enable):
        check(lib().dip_plan_set_timing(self.h, int(bool(enable))))

    def get_timing(self):
        """{'fprop'|'dgrad'|'wgrad': (ms, algorithmic flops, launches)} since the last call (syncs on the events)."""
        ms, fl, n = (ctypes.c_double * 3)(), (ctypes.c_double * 3)(), (ctypes.c_int * 3)()
        check(lib().dip_plan_get_timing(self.h, ms, fl, n))
        return {k: (ms[i], fl[i], n[i]) for i, k in enumerate(("fprop", "dgrad", "wgrad"))}

    def get_timing_records(self, max_records=65536):
        """[(class 0 fprop | 1 dgrad | 2 wgrad, algorithmic flops, ms)] per tensor-core launch since the last call."""
        cls, fl, ms = (ctypes.c_int * max_records)(), (ctypes.c_double * max_records)(), (ctypes.c_double * max_records)()
        n = lib().dip_plan_get_timing_records(self.h, max_records, cls, fl, ms)
        if n < 0:
            check(n)
        return [(cls[i], fl[i], ms[i]) for i in range(n)]

    def num_launches(self):
        a, b = ctypes.c_int(), ctypes.c_int()
        lib().dip_plan_num_launches(self.h, ctypes.byref(a), ctypes.byref(b))
        return a.value, b.value


class FusedAdam:
    """torch.optim.Adam(params, lr).step() as one multi-tensor kernel (dip_adam_* in include/dip.h)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8):
        self.params = list(params)
        self.lr, self.betas, self.eps = lr, betas, eps
        self.step_count = 0
        dev = self.params[0].device
        numel = [p.numel() for p in self.params]
        self.m_flat = torch.zeros(sum(numel), dtype=torch.float32, device=dev)
        self.v_flat = torch.zeros(sum(numel), dtype=torch.float32, device=dev)
        self.m, self.v = [], []
        o = 0
        for n in numel:
            self.m.append(self.m_flat[o:o + n])
            self.v.append(self.v_flat[o:o + n])
            o += n
        arr = (ctypes.c_longlong * len(numel))(*numel)
        h = ctypes.c_void_p()
        with torch.cuda.device(dev):
            check(lib().dip_adam_create(len(numel), arr, ctypes.byref(h)))
        self.h = h
        self._key = None

    def __del__(self):
        try:
            if getattr(self, "h", None) is not None and _lib is not None:
                _lib.dip_adam_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def zero_grad(self):
        for p in self.params:
            p.grad = None

    def _bind(self, grads):
        key = (tuple(p.data_ptr() for p in self.params), tuple(g.data_ptr() for g in grads))
        if key != self._key:
            with torch.cuda.device(self.params[0].device):
                check(lib().dip_adam_bind(self.h, _ptr_array(self.params), _ptr_array(grads), _ptr_array(self.m),
                                          _ptr_array(self.v)))
            self._key = key

    def step(self):
        grads = [p.grad for p in self.params]
        if any(g is None for g in grads):
            raise RuntimeError("FusedAdam.step: a parameter has no gradient")
        self._bind(grads)
        self.step_count += 1
        with torch.cuda.device(self.params[0].device):
            check(lib().dip_adam_step(self.h, self.lr, self.betas[0], self.betas[1], self.eps, self.step_count,
                                      _stream()))


class Tracker:
    """State of the denoising closure (denoising.ipynb c10:8-52) that run_iterations(track=...) keeps on the device: the
    EMA `out_avg`, the parameter snapshot (`last_net`, flat in the Adam tensors' order like FusedAdam.m_flat) and the
    back-tracking state.  gt: the clean image (psnr_gt / psnr_gt_sm; NaN without it).  Defaults are c10's."""

    def __init__(self, adam, out_shape, gt=None, exp_weight=0.99, show_every=100, backtrack_db=5.0):
        dev = adam.params[0].device
        self.adam = adam
        self.gt = None if gt is None else gt.detach().to(device=dev, dtype=torch.float32).contiguous()
        if self.gt is not None and tuple(self.gt.shape) != tuple(out_shape):
            raise ValueError("dip-b200: Tracker gt has shape %s, the output %s" % (tuple(self.gt.shape), tuple(out_shape)))
        self.exp_weight, self.show_every, self.backtrack_db = float(exp_weight), int(show_every), float(backtrack_db)
        self.out_avg = torch.zeros(out_shape, dtype=torch.float32, device=dev)
        self.snapshot = torch.zeros(adam.m_flat.numel(), dtype=torch.float32, device=dev)
        self.state = torch.zeros(lib().dip_track_state_bytes(), dtype=torch.uint8, device=dev)

    def reset(self):
        """back to the notebook's initial globals: i = 0, out_avg = None, last_net = None, psrn_noisy_last = 0"""
        self.state.zero_()

    def _state(self):
        s = self.state.cpu()
        return s[:8].view(torch.float64).item(), s[8:].view(torch.int32).tolist()   # TrackState (kernels.cuh)

    @property
    def i(self):
        return self._state()[1][0]

    @property
    def fallbacks(self):
        return self._state()[1][4]

    @property
    def psnr_last(self):
        return self._state()[0]

    def struct(self, records):
        return Track(_ptr(self.gt).value, self.out_avg.data_ptr(), self.snapshot.data_ptr(), self.state.data_ptr(),
                     records.data_ptr(), self.exp_weight, self.show_every, self.backtrack_db)


def run_iterations(plan, adam, z0, target, mask, sigma, seed, iters, lr, out=None, loss_hist=None, track=None,
                   records=None):
    """Closure-free device loop (dip_run_iterations): noise -> forward -> MSE -> backward -> Adam, `iters` times.
    The device loop's Adam step uses torch's default betas and eps; an optimiser with others is refused, not stepped
    with the defaults.  track: a Tracker of `adam`, which then needs `records`, an fp64 CUDA tensor of iters x 6
    (dip_run_iterations_tracked)."""
    if tuple(adam.betas) != (0.9, 0.999):
        raise ValueError("dip-b200: run_iterations steps Adam with betas (0.9, 0.999); adam.betas is %r" % (adam.betas,))
    if adam.eps != 1e-8:
        raise ValueError("dip-b200: run_iterations steps Adam with eps 1e-8; adam.eps is %r" % (adam.eps,))
    tr = None
    if track is not None:
        if track.adam is not adam:
            raise ValueError("dip-b200: run_iterations: the Tracker belongs to another optimiser")
        if (records is None or not records.is_cuda or records.dtype != torch.float64 or not records.is_contiguous()
                or records.numel() < RECORD * iters):
            raise ValueError("dip-b200: run_iterations(track=...) needs records, a contiguous fp64 CUDA tensor of >= %d x %d"
                             % (iters, RECORD))
        tr = ctypes.byref(track.struct(records))
    elif records is not None:
        raise ValueError("dip-b200: run_iterations: records without a Tracker")
    with torch.cuda.device(plan.device):
        check(lib().dip_run_iterations_tracked(plan.h, adam.h, _ptr(z0), _ptr(target), _ptr(mask), float(sigma), int(seed),
                                               adam.step_count, int(iters), float(lr), _ptr(out), _ptr(loss_hist), tr,
                                               _stream()))
    adam.step_count += iters


# ------------------------------------------------------------------------------------------------ downsampler
def down_out_size(n, K, factor, pad):
    return (n + 2 * pad - K) // factor + 1 if n + 2 * pad >= K else 0


def lanczos_down_fwd(x, kern, factor, pad):
    """x: (1|N) x C x H x W CUDA fp32 planes, kern: K x K CUDA fp32 taps -> planes downsampled by `factor`."""
    assert x.is_cuda and x.dtype == torch.float32 and kern.is_cuda and kern.dtype == torch.float32
    x = x.contiguous()
    kern = kern.contiguous()
    n, c, H, W = x.shape
    K = int(kern.shape[-1])
    y = torch.empty((n, c, down_out_size(H, K, factor, pad), down_out_size(W, K, factor, pad)), dtype=torch.float32,
                    device=x.device)
    with torch.cuda.device(x.device):
        check(lib().dip_lanczos_down_fwd(_ptr(x), n * c, H, W, _ptr(kern), K, int(factor), int(pad), _ptr(y), _stream()))
    return y


def lanczos_down_bwd(dy, kern, factor, pad, H, W):
    assert dy.is_cuda and dy.dtype == torch.float32
    dy = dy.contiguous()
    kern = kern.contiguous()
    n, c = dy.shape[0], dy.shape[1]
    K = int(kern.shape[-1])
    dx = torch.empty((n, c, H, W), dtype=torch.float32, device=dy.device)
    with torch.cuda.device(dy.device):
        check(lib().dip_lanczos_down_bwd(_ptr(dy), n * c, H, W, _ptr(kern), K, int(factor), int(pad), _ptr(dx), _stream()))
    return dx


# ------------------------------------------------------------------------------------------------ single ops (tests)
_scratch = {}


def _get_scratch(dev):
    key = str(dev)
    if key not in _scratch:
        _scratch[key] = torch.empty(lib().dip_op_scratch_bytes(), dtype=torch.uint8, device=dev)
    return _scratch[key]


def op_conv_fprop(a_nhwc, w, bias, k, stride, offx, offy, d_h, d_w, rot=0, stats=None, precision=PRECISION_TF32):
    a_h, a_w, a_c = a_nhwc.shape
    N, C = w.shape[0], w.shape[1]
    d = torch.empty((d_h, d_w, N), dtype=torch.float32, device=a_nhwc.device)
    check(lib().dip_op_conv_fprop(_ptr(a_nhwc), a_h, a_w, a_c, _ptr(w), _ptr(bias), N, C, k, stride, offx, offy, rot,
                                  _ptr(d), d_h, d_w, _ptr(stats), precision, _ptr(_get_scratch(a_nhwc.device)),
                                  _stream()))
    return d


def op_conv_dgrad(dy_nhwc, w, k, dx_h, dx_w, rot=0, precision=PRECISION_TF32):
    dy_h, dy_w, n = dy_nhwc.shape
    N, C = w.shape[0], w.shape[1]
    assert n == N
    dx = torch.empty((dx_h, dx_w, C), dtype=torch.float32, device=dy_nhwc.device)
    check(lib().dip_op_conv_dgrad(_ptr(dy_nhwc), dy_h, dy_w, _ptr(w), N, C, k, rot, _ptr(dx), dx_h, dx_w, precision,
                                  _ptr(_get_scratch(dy_nhwc.device)), _stream()))
    return dx


def op_conv_dgrad_s2(dy_nhwc, w, rot=0, precision=PRECISION_TF32):
    """Input gradient of a 3x3 stride-2 conv (4 sub-pixel phases): dy [h][w][128] -> dx [(2h+2)][(2w+2)][C]."""
    dy_h, dy_w, n = dy_nhwc.shape
    N, C = w.shape[0], w.shape[1]
    assert n == N
    dx = torch.full((2 * dy_h + 2, 2 * dy_w + 2, C), float("nan"), dtype=torch.float32, device=dy_nhwc.device)
    check(lib().dip_op_conv_dgrad_s2(_ptr(dy_nhwc), dy_h, dy_w, _ptr(w), N, C, rot, _ptr(dx), precision,
                                     _ptr(_get_scratch(dy_nhwc.device)), _stream()))
    return dx


def op_conv_wgrad(dy_nhwc, a_nhwc, C, k, stride, offx, offy, rot=0, precision=PRECISION_TF32):
    dy_h, dy_w, N = dy_nhwc.shape
    a_h, a_w, a_c = a_nhwc.shape
    dw = torch.empty((N, C, k, k), dtype=torch.float32, device=dy_nhwc.device)
    check(lib().dip_op_conv_wgrad(_ptr(dy_nhwc), dy_h, dy_w, _ptr(a_nhwc), a_h, a_w, a_c, N, C, k, stride, offx, offy,
                                  rot, _ptr(dw), precision, _ptr(_get_scratch(dy_nhwc.device)), _stream()))
    return dw
