#!/usr/bin/env python
"""bench.py -- deep-image-prior hot path on H100: optimisation iterations/sec, 512x512 skip-net denoising.

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--dump-outputs DIR]
  python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py --gpus N --steps K --warmup W

A "step" is one optimisation iteration of BASELINE.json configs[1] (denoising F16-sized 512x512, skip[128x5], fp32):
  z = z0 + N(0,1)/30  ->  out = net(z)  ->  MSE(out, noisy target)  ->  backward  ->  Adam(lr 0.01) step.
One independent image per GPU (weak scaling, no data-path collective; NCCL only for barriers and the result gather).

Order of the run (our arm), all on the device clock (CUDA events), max over ranks:
  1. W warm-up steps, then ONE FULL IMAGE = 2000 iterations (BASELINE.json configs[0]/[1] budget, ~6 s): `image_run`
     and `images_per_sec` are MEASURED over it, with nvidia-smi clocks sampled throughout (sustained clocks);
  2. immediately after, the K steps asked for -> `value` / `ms_per_step` (clocks already in their sustained
     state, inputs resident in HBM, closure-free device runner dip_run_iterations); --dump-outputs DIR writes what these
     steps computed (out.npy, loss_hist.npy, params.npy);
  3. a short eager pass with CUDA events around every launch -> `roofline*` (algorithmic FLOPs or bytes / device time);
  4. `e2e`: utils.optimize('adam', params, closure, LR, n) with the notebook's closure (on-device noise.normal_() like
     denoising.ipynb c10:12-13, the step's input copied host(pinned)->device and the loss read back inside the region);
     `e2e_verbatim_closure`: the same with the verbatim c10 closure (EMA, 3 x PSNR read-backs, parameter snapshot);
  5. `gpu_library_baseline`: the SAME module tree executed by stock torch.cuda + cuDNN (cudnn.benchmark, TF32 default),
     lean closure -- the reference's own GPU path on the same GPU (BASELINE.md 3.4);
  6. rank 0, N=1: `cpu_baseline` = the reference arm below on a bounded sample.
--impl reference: the reference's CPU implementation of the same step on the host cores: the UNMODIFIED reference from
  oracle/_ref (copied by oracle/make_ref.py; kind "reference") when present, else the oracle port (kind "port").
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.join(ROOT, "deep-image-prior_b200")
REF_COPY = os.path.join(ROOT, "oracle", "_ref")

H = W = 512
IN_CH, OUT_CH = 32, 3
SIGMA_REG = 1.0 / 30.0
LR = 0.01
ITERS_PER_IMAGE = 2000           # BASELINE.json configs[0]/[1]
ALG_GFLOP_PER_ITER = 460.07      # SURVEY.md section 6 (2*M*N*K over the 26 convs, fwd+dgrad+wgrad)
# dram__bytes_read.sum + dram__bytes_write.sum of the dominant launches, when a capture is committed under profiles/
TRAFFIC = json.load(open(os.path.join(ROOT, "profiles", "traffic.json"))) if os.path.exists(
    os.path.join(ROOT, "profiles", "traffic.json")) else {}
METRIC = "optimisation iterations/sec (512x512 skip-net denoising, sum over independent images)"
WORKLOAD = ("denoise 512x512 skip[128x5] in32 out3 bilinear, noise+fwd+MSE+bwd+Adam per step (BASELINE.json configs[1]); "
            "one independent image per GPU")

HBM_NAMES = ["k_input_pad", "k_noise", "k_skinny_fwd", "k_bn_act_write", "k_bn_act_head", "k_cat_stats", "k_cat_write",
             "k_bn_bwd_reduce", "k_bn_bwd_apply", "k_cat_bwd_reduce", "k_cat_bwd_apply", "k_upadj", "k_skinny_bwd", "k_mse",
             "k_adam", "k_head_dlogit", "k_down_fwd", "k_down_bwd", "k_pack_table", "k_wgrad_reduce"]


def load_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        return json.load(open(p)), "measured (MEASURED_PEAKS.json)"
    # NVIDIA's H100 SXM data sheet (dense BF16; TF32 is half of it) -- an upper bound, not a rate this card has been seen to reach
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0}, "H100 SXM data sheet"


class ClockSampler:
    """nvidia-smi clocks / throttle reasons, one row every 20 ms with its arrival time, for the whole GPU section;
    window(t0, t1) summarises the rows that fell inside a timed region."""

    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")
    NAMES = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]

    def __init__(self, index):
        self.index, self.rows, self.proc = index, [], None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.Q,
                                          "--format=csv,noheader,nounits", "-lms", "20"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append((time.time(), [x.strip() for x in line.split(",")]))

    def stop(self):
        if self.proc is not None:
            self.proc.terminate()
            try:
                self.proc.wait(timeout=5)
            except Exception:
                pass

    def window(self, t0, t1):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "samples": 0, "reasons": ["nvidia-smi unavailable"]}
        sm, mx, pw, reasons = [], [], [], set()
        for t, r in list(self.rows):
            if t < t0 or t > t1 or len(r) < 8:
                continue
            try:
                sm.append(float(r[1]))
                mx.append(float(r[2]))
                pw.append(float(r[3]))
            except ValueError:
                continue
            for n, v in zip(self.NAMES, r[4:8]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_min_mhz": sm[0] if sm else None,
                "sm_max_mhz": max(mx) if mx else None, "power_w_max": max(pw) if pw else None, "samples": len(sm),
                "reasons": sorted(reasons)}


def make_problem(torch, seed):
    """Synthetic inputs of the BASELINE shape (no dataset on the box): z0 ~ U[0,0.1), target = clip(img + N(0,25/255))."""
    g = torch.Generator().manual_seed(1000 + seed)
    z0 = torch.rand(1, IN_CH, H, W, generator=g) * 0.1
    clean = torch.rand(1, OUT_CH, H // 8, W // 8, generator=g)
    clean = torch.nn.functional.interpolate(clean, size=(H, W), mode="bilinear", align_corners=False)
    target = (clean + torch.randn(clean.shape, generator=g) * (25.0 / 255.0)).clamp(0, 1)
    return z0, clean, target


# ------------------------------------------------------------------------------------------------ reference arm (CPU)
class CpuReference:
    """The reference's per-iteration path on torch-CPU: the unmodified reference (oracle/_ref) or the oracle port."""

    def __init__(self, torch):
        self.torch = torch
        sys.path.insert(0, ROOT)
        self.kind = "reference" if os.path.isdir(os.path.join(REF_COPY, "models")) else "port"
        if self.kind == "reference":
            from oracle import ref_harness
            ref_harness._install_shims()
            sys.path.insert(0, REF_COPY)               # `models` / `utils` = the reference's own packages in THIS process
            import models as ref_models
            import utils.common_utils as ref_cu
            assert os.path.realpath(os.path.dirname(ref_models.__file__)).startswith(os.path.realpath(REF_COPY))
            self.models, self.cu = ref_models, ref_cu
            self.detail = "oracle/_ref: the UNMODIFIED reference (models.get_net + the lean closure of denoising.ipynb c10 + utils.optimize) on torch-CPU"
        else:
            from oracle import dip_oracle
            self.O = dip_oracle
            self.detail = "oracle/dip_oracle.py: port of the reference's graph on torch-CPU (oracle/_ref not present)"

    def setup(self, h, w):
        torch = self.torch
        self.z0 = torch.rand(1, IN_CH, h, w) * 0.1
        self.target = torch.rand(1, OUT_CH, h, w)
        if self.kind == "reference":
            torch.manual_seed(0)
            self.net = self.models.get_net(IN_CH, 'skip', 'reflection', skip_n33d=128, skip_n33u=128, skip_n11=4, num_scales=5,
                                           upsample_mode='bilinear').type(torch.FloatTensor)
            self.mse = torch.nn.MSELoss()
            self.noise = self.z0.clone()
        else:
            self.cfg = self.O.SkipConfig(upsample_mode="bilinear")
            self.params = self.O.init_params(self.cfg, seed=0)
            self.opt = self.O.Adam(self.params, LR)

    def run(self, n):
        """n iterations; returns seconds."""
        torch = self.torch
        t0 = time.perf_counter()
        if self.kind == "reference":
            def closure():
                net_input = self.z0 + (self.noise.normal_() * SIGMA_REG)
                out = self.net(net_input)
                total_loss = self.mse(out, self.target)
                total_loss.backward()
                total_loss.item()
                return total_loss
            import contextlib
            import io
            with contextlib.redirect_stdout(io.StringIO()):     # optimize() prints "Starting optimization with ADAM"
                self.cu.optimize('adam', self.cu.get_params('net', self.net, self.z0), closure, LR, n)
        else:
            for _ in range(n):
                z = self.z0 + torch.randn(self.z0.shape) * SIGMA_REG
                loss = self.O.mse_loss(self.O.skip_forward(self.params, z, self.cfg), self.target)
                self.opt.step(torch.autograd.grad(loss, self.params))
                loss.item()
        return time.perf_counter() - t0


def best_cpu_threads(torch, ref):
    """torch-CPU gets slower, not faster, when all 100+ logical cores of the GPU box are used (MKL-DNN oversubscription on
    a shared host): pick the thread count that serves the reference best on a quarter-size probe; `cores` reports it."""
    cores = os.cpu_count() or 1
    cands = sorted(set(c for c in (8, 16, 32, 64, cores) if c <= cores))
    ref.setup(256, 256)
    best, best_t = cands[0], None
    for c in cands:
        torch.set_num_threads(c)
        ref.run(1)                                  # warms the thread pool
        dt = ref.run(1)
        if best_t is None or dt < best_t:
            best, best_t = c, dt
    return best


def run_reference(args):
    import torch
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    ref = CpuReference(torch)
    cores = best_cpu_threads(torch, ref)
    torch.set_num_threads(cores)
    budget_s = float(os.environ.get("DIP_REF_BUDGET_S", "150"))
    t0 = time.perf_counter()
    ref.setup(H, W)
    s_per = ref.run(1)                              # first full-size iteration: warm-up, also sizes the bounded sample
    warm = max(0, min(args.warmup, 3) - 1)
    steps = max(1, min(args.steps, int((budget_s - (time.perf_counter() - t0)) / s_per) - warm))
    if warm:
        ref.run(warm)
    secs = ref.run(steps)
    its = steps / secs
    sample = ("%d timed iterations (of %d requested) after %d warm-up, full 512x512 workload, %d threads (best of a probe over "
              "{8,16,32,64,all}; host has %d logical cores)" % (steps, args.steps, warm + 1, cores, os.cpu_count() or 1))
    line = {"impl": "reference", "metric": METRIC, "value": its, "unit": "it/s", "n_gpus": args.gpus, "steps": steps,
            "steps_requested": args.steps, "warmup": warm + 1, "ms_per_step": 1000.0 * secs / steps, "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None, "dtype": "fp32", "data": "synthetic",
            "config": {"workload": WORKLOAD, "impl_detail": ref.detail},
            "cpu_baseline": {"value": its, "unit": "it/s", "cores": cores, "kind": ref.kind, "sample": sample},
            "e2e": {"value": its, "unit": "it/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "gpu_launches": 0}
    print(json.dumps(line), flush=True)


# ------------------------------------------------------------------------------------------------ our arm (GPU)
def run_ours(args):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, PKG)
    import numpy as np
    import torch
    import torch.distributed as dist
    import dip_engine as de
    import multi_gpu as mg
    import models
    import contextlib
    import io
    from utils.common_utils import get_params
    from utils.common_utils import optimize as _optimize

    def optimize(*a):                       # utils.optimize prints "Starting optimization with ADAM" like the reference does:
        with contextlib.redirect_stdout(io.StringIO()):   # stdout must stay the one JSON line
            _optimize(*a)

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world != args.gpus and world == 1 and args.gpus > 1:
        raise SystemExit("launch with torch.distributed.run --nproc-per-node %d" % args.gpus)
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)   # NCCL_DEBUG is left as the caller set it
    peaks, peak_src = load_peaks()
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()                                  # before any warm-up: every window below has samples

    # ---- build the network through the public API (same seeds on every rank; different image per rank)
    dtype = torch.cuda.FloatTensor
    torch.manual_seed(0)
    net = models.get_net(IN_CH, "skip", "reflection", skip_n33d=128, skip_n33u=128, skip_n11=4, num_scales=5,
                         upsample_mode="bilinear").type(dtype)
    z0_h, clean_h, target_h = make_problem(torch, rank)
    z0, target = z0_h.to(dev), target_h.to(dev)
    params = [p for p in net.parameters()]
    opt = de.FusedAdam(params, lr=LR)
    mse = torch.nn.MSELoss().type(dtype)

    def api_step(z_dev):
        opt.zero_grad()
        out = net(z_dev)
        loss = mse(out, target)
        loss.backward()
        opt.step()
        return loss

    api_step(z0)    # creates the plan, binds parameters / gradients, attaches .grad views
    torch.cuda.synchronize()
    plan = list(net._dip_plans.values())[0]
    opt._bind([p.grad for p in params])
    out_buf = torch.empty(1, OUT_CH, H, W, device=dev)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def device_steps(n, hist=None):
        de.run_iterations(plan, opt, z0, target, None, SIGMA_REG, 1234 + rank, n, LR, out=out_buf, loss_hist=hist)

    def timed(fn):
        """fn() bracketed by barrier + synchronize on both sides, CUDA events on the launching stream; returns
        (ms max over ranks, (wall t0, wall t1) of this rank for the clock window)."""
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        barrier()
        w0 = time.time()
        e0.record()
        fn()
        e1.record()
        barrier()
        w1 = time.time()
        return mg.max_over_ranks(e0.elapsed_time(e1), device=dev), (w0, w1)

    # ---- 1. warm-up, then one full image (2000 iterations) ----------------------------------------------------------
    warm = max(args.warmup, 3)
    device_steps(warm)
    img_hist = torch.zeros(ITERS_PER_IMAGE, dtype=torch.float64, device=dev)
    img_ms, img_win = timed(lambda: device_steps(ITERS_PER_IMAGE, img_hist))
    with torch.no_grad():
        psnr_img = 10 * np.log10(1.0 / float(((out_buf.cpu() - clean_h) ** 2).mean()))
    # ---- 2. `value`: the K steps asked for, right behind the image (sustained clocks) -------------------
    hist = torch.zeros(args.steps, dtype=torch.float64, device=dev)
    ms, val_win = timed(lambda: device_steps(args.steps, hist))
    value = mg.aggregate_rate(args.steps, ms / 1000.0, world)
    if args.dump_outputs and rank == 0:
        # what the timed steps hand back: the network output of the last step, the loss of every step and the parameters
        # after the last Adam update (float32 / float64, ~13 MB); the inputs are seeded, so two builds compare value by value
        os.makedirs(args.dump_outputs, exist_ok=True)
        np.save(os.path.join(args.dump_outputs, "out.npy"), out_buf.float().cpu().numpy())
        np.save(os.path.join(args.dump_outputs, "loss_hist.npy"), hist.cpu().numpy())
        np.save(os.path.join(args.dump_outputs, "params.npy"),
                torch.cat([p.detach().reshape(-1) for p in params]).float().cpu().numpy())

    # ---- 3. roofline pass: CUDA events around every launch of a short eager pass (graphs cannot be event-bracketed) --
    roof_steps = min(args.steps, 10)
    os.environ["DIP_NO_SIDE"] = "1"       # kernels timed one at a time (the graph overlaps side streams)
    plan.set_timing(True)
    device_steps(roof_steps)
    torch.cuda.synchronize()
    records = plan.get_timing_records()
    plan.set_timing(False)
    os.environ.pop("DIP_NO_SIDE", None)
    fwd_l, bwd_l = plan.num_launches()
    launches_per_step = fwd_l + bwd_l + 3      # + noise, mse, adam

    # ---- 4. e2e: utils.optimize() with the notebook closure, host input + loss read-back in the timed region --------
    z_pinned = z0_h.pin_memory()
    noise = z0.detach().clone()
    last = {"loss": 0.0}
    # every step's input crosses PCIe inside the timed region (33.5 MB, ~0.6 ms): the copy for step i+1 is issued on a copy
    # stream while step i computes (double-buffered device input), as any input pipeline would do
    zbuf = [torch.empty_like(z0), torch.empty_like(z0)]
    copy_stream = torch.cuda.Stream()
    ready = [torch.cuda.Event(), torch.cuda.Event()]
    consumed = [torch.cuda.Event(), torch.cuda.Event()]
    pipe = {"i": 0}
    # the step's loss is read back EVERY step, through a pinned buffer and one step late: the copy of step i is issued
    # behind step i's kernels and consumed while step i+1 runs, so the host never stalls the device on .item()
    loss_pin = [torch.zeros(1).pin_memory(), torch.zeros(1).pin_memory()]
    loss_ev = [torch.cuda.Event(), torch.cuda.Event()]

    def prefetch(i):
        b = i % 2
        with torch.cuda.stream(copy_stream):
            copy_stream.wait_event(consumed[b])                # the step that last read this buffer has finished
            zbuf[b].copy_(z_pinned, non_blocking=True)         # H2D: the step's input
            ready[b].record(copy_stream)

    def pipe_reset():
        torch.cuda.synchronize()
        for b in range(2):
            consumed[b].record()
        pipe["i"] = 0
        prefetch(0)

    def lean_closure():                      # denoising.ipynb c10:8-24 without the logging
        i = pipe["i"]
        b = i % 2
        torch.cuda.current_stream().wait_event(ready[b])
        net_input = zbuf[b] + (noise.normal_() * SIGMA_REG)                   # c10:12-13, device RNG
        consumed[b].record()
        prefetch(i + 1)
        pipe["i"] = i + 1
        out = net(net_input)
        total_loss = mse(out, target)
        total_loss.backward()
        loss_pin[b].copy_(total_loss.detach().reshape(1), non_blocking=True)  # D2H: the step's loss
        loss_ev[b].record()
        if i > 0:
            loss_ev[1 - b].synchronize()                                      # the previous step's loss has landed
            last["loss"] = float(loss_pin[1 - b][0])
        return total_loss

    e2e_steps = max(args.steps, 200)
    pipe_reset()
    optimize("adam", get_params("net", net, z0), lean_closure, LR, 5)

    def e2e_run():
        prefetch(pipe["i"])          # (re-issued inside the timed region: the first step's H2D is timed too)
        optimize("adam", get_params("net", net, z0), lean_closure, LR, e2e_steps)
    e2e_ms, _ = timed(e2e_run)
    e2e_value = mg.aggregate_rate(e2e_steps, e2e_ms / 1000.0, world)

    # verbatim closure of denoising.ipynb c10 (SURVEY.md 8f.1): EMA, three PSNR read-backs, last_net snapshot
    img_np, img_noisy_np = clean_h.numpy()[0], target_h.numpy()[0]
    st = {"i": 0, "out_avg": None, "last_net": None, "psrn_noisy_last": 0}

    def psnr_np(a, b):
        return 10 * np.log10(1.0 / np.mean((a.astype(np.float64) - b) ** 2))

    def verbatim_closure():
        net_input = z0 + (noise.normal_() * SIGMA_REG)
        out = net(net_input)
        st["out_avg"] = out.detach() if st["out_avg"] is None else st["out_avg"] * 0.99 + out.detach() * 0.01
        total_loss = mse(out, target)
        total_loss.backward()
        psrn_noisy = psnr_np(img_noisy_np, out.detach().cpu().numpy()[0])
        psnr_np(img_np, out.detach().cpu().numpy()[0])
        psnr_np(img_np, st["out_avg"].detach().cpu().numpy()[0])
        total_loss.item()
        if st["i"] % 100:
            if psrn_noisy - st["psrn_noisy_last"] < -5:
                for new_param, net_param in zip(st["last_net"], net.parameters()):
                    net_param.data.copy_(new_param.cuda())
                return total_loss * 0
            st["last_net"] = [x.detach().cpu() for x in net.parameters()]
            st["psrn_noisy_last"] = psrn_noisy
        st["i"] += 1
        return total_loss

    vb_steps = 50
    optimize("adam", get_params("net", net, z0), verbatim_closure, LR, 3)
    vb_ms, _ = timed(lambda: optimize("adam", get_params("net", net, z0), verbatim_closure, LR, vb_steps))
    vb_value = mg.aggregate_rate(vb_steps, vb_ms / 1000.0, world)

    # the same closure logic with device-side metrics (utils/fast_closure.py): one 32-byte read-back per iteration
    from utils.fast_closure import DenoisingClosure
    fast = DenoisingClosure(net, z0, target, clean_h.to(dev), reg_noise_std=SIGMA_REG, exp_weight=0.99, show_every=100, mse=mse)
    fv_steps = max(args.steps, 200)
    optimize("adam", get_params("net", net, z0), fast, LR, 5)
    fv_ms, _ = timed(lambda: optimize("adam", get_params("net", net, z0), fast, LR, fv_steps))
    fv_value = mg.aggregate_rate(fv_steps, fv_ms / 1000.0, world)

    # ---- 5. the reference's own GPU path: same module tree on stock torch.cuda + cuDNN ------------------------------
    lib_value = None
    if rank == 0:
        torch.backends.cudnn.enabled = True
        torch.backends.cudnn.benchmark = True          # denoising.ipynb c3:17-18
        torch.manual_seed(0)
        net_t = models.get_net(IN_CH, "skip", "reflection", skip_n33d=128, skip_n33u=128, skip_n11=4, num_scales=5,
                               upsample_mode="bilinear").type(dtype)
        net_t._dip_spec, net_t._dip_why = None, "bench.py gpu_library_baseline: stock torch modules requested"
        models.allow_torch_execution(True)
        try:
            topt = torch.optim.Adam(net_t.parameters(), lr=LR)
            noise_t = z0.detach().clone()

            def lib_steps(n):
                for _ in range(n):
                    topt.zero_grad()
                    out = net_t(z0 + (noise_t.normal_() * SIGMA_REG))
                    mse(out, target).backward()
                    topt.step()
            lib_steps(10)                               # cudnn.benchmark autotuning + allocator warm-up
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            n_lib = 50
            e0.record()
            lib_steps(n_lib)
            e1.record()
            torch.cuda.synchronize()
            lib_value = n_lib / (e0.elapsed_time(e1) / 1000.0)
        finally:
            models.allow_torch_execution(False)
        del net_t, topt
    if world > 1:
        dist.barrier()

    # ---- 6. BASELINE configs[2]: super-resolution x4 (1024^2 net output -> 256^2 through the Lanczos-2 operator), runner,
    #         in the default tf32 mode and in bf16 (wgmma on bf16 operands) -- single GPU, rank 0 only
    sr_cfg = None
    if rank == 0 and world == 1:
        del fast
        torch.cuda.empty_cache()
        try:
            sr_cfg = bench_sr_config(torch, de, models, peaks, dev)
        except Exception as e:      # the headline line must still come out
            sr_cfg = {"error": repr(e)[:300]}

    # ---- result record per rank (the only data collective of the job)
    recs = mg.gather_records([psnr_img, float(img_hist[-1].item()), ITERS_PER_IMAGE / (img_ms / 1000.0)], device=dev)
    sampler.stop()

    if rank == 0:
        tf32_sust = peaks.get("bf16_tflops_sustained", peaks["bf16_tflops"]) / 2.0
        tf32_burst = peaks["bf16_tflops"] / 2.0
        step_ms = ms / args.steps

        def agg(pred):
            sel = [r for r in records if pred(r)]
            ms_, fl_ = sum(r[2] for r in sel), sum(r[1] for r in sel)
            return ms_, fl_, len(sel)

        def tensor_roof(name, pred, extra=None):
            ms_, fl_, n_ = agg(pred)
            ach = fl_ / (ms_ / 1000.0) / 1e12 if ms_ > 0 else 0.0
            d = {"kernel": name, "bound": "tensor", "achieved": ach, "peak": tf32_burst, "unit": "TFLOP/s",
                 "frac": ach / tf32_burst, "peak_sustained": tf32_sust, "frac_vs_sustained": ach / tf32_sust,
                 "launches_per_step": n_ // max(roof_steps, 1), "ms_per_step": ms_ / roof_steps,
                 "share_of_step": (ms_ / roof_steps) / step_ms,
                 "algorithmic_flops_per_step": fl_ / roof_steps}
            d.update(extra or {})
            return d

        def hbm_roof(name, pred, extra=None):
            ms_, by_, n_ = agg(pred)
            ach = by_ / (ms_ / 1000.0) / 1e9 if ms_ > 0 else 0.0
            d = {"kernel": name, "bound": "hbm", "achieved": ach, "peak": peaks["hbm_gbs"], "unit": "GB/s",
                 "frac": ach / peaks["hbm_gbs"], "launches_per_step": n_ // max(roof_steps, 1),
                 "ms_per_step": ms_ / roof_steps, "share_of_step": (ms_ / roof_steps) / step_ms,
                 "algorithmic_bytes_per_step": by_ / roof_steps}
            d.update(extra or {})
            return d

        note = ("peak = tf32 dense = 1/2 of the bf16 rate (%s); the kernels are timed alone in a ~30 ms pass; "
                "peak_sustained = 1/2 of the sustained bf16 rate where one was measured" % peak_src)
        roof = tensor_roof("tc_conv_kernel (wgmma tf32 implicit GEMM): ALL fprop + dgrad launches of a step",
                           lambda r: r[0] in (0, 1),
                           {"peak_note": note, "traffic": TRAFFIC.get("tc_conv_dominant"),
                            "traffic_note": "dram read+write of the dominant launch (level-0 3x3 up conv fprop) from profiles/; null until captured",
                            "timed": "CUDA events around every launch in a %d-step eager pass right after the timed region "
                                     "(side streams off so that kernels run alone)" % roof_steps})
        big = max(r[1] for r in records if r[0] == 0)
        by_kernel = {}
        for kid, nm in enumerate(HBM_NAMES):
            sel = [r for r in records if r[0] >= 16 and (r[0] - 16) // 8 == kid]
            if sel:
                ms_, by_ = sum(r[2] for r in sel), sum(r[1] for r in sel)
                by_kernel[nm] = {"GB/s": by_ / (ms_ / 1000.0) / 1e9, "us_per_step": 1000.0 * ms_ / roof_steps,
                                 "launches_per_step": len(sel) // roof_steps}
        hbm_big = max((r[1] for r in records if r[0] == 16 + 8 * 8), default=0.0)     # bn_bwd_apply, plain source
        line = {
            "metric": METRIC, "value": value, "unit": "it/s", "n_gpus": world, "steps": args.steps, "warmup": warm,
            "ms_per_step": step_ms, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "fp32 storage; tf32 tensor-core multiplies with fp32 accumulate in the convs (cuDNN's default fp32 mode)",
            "data": "synthetic",
            "config": {"workload": WORKLOAD, "iters_per_image": ITERS_PER_IMAGE,
                       "l2": "per-step working set 2.5 GB >> 126 MB L2 (inputs larger than L2, no flush needed)",
                       "precision": "tf32", "peaks": peak_src,
                       "order": "warm-up, one full 2000-iteration image (image_run), then the K timed steps (value)"},
            "image_run": {"iters": ITERS_PER_IMAGE, "seconds": img_ms / 1000.0,
                          "it_per_s": world * ITERS_PER_IMAGE / (img_ms / 1000.0), "clocks": sampler.window(*img_win),
                          "final_loss": float(img_hist[-1].item()), "psnr_vs_clean_rank0": psnr_img,
                          "note": "measured, not extrapolated: every GPU optimises one whole image"},
            "images_per_sec": world / (img_ms / 1000.0),
            "clocks": sampler.window(*val_win),
            "e2e": {"value": e2e_value, "unit": "it/s", "h2d_bytes_per_step": int(z0.numel() * 4), "d2h_bytes_per_step": 4,
                    "steps": e2e_steps, "last_loss": last["loss"],
                    "api": "utils.optimize('adam', get_params('net', net, z), closure, LR, n) on models.get_net(...).type(cuda); "
                           "closure = denoising.ipynb c10 without logging: input H2D from pinned memory (prefetched one step ahead), "
                           "noise.normal_() on the device, net(), MSELoss, backward(), the loss copied to pinned host memory every "
                           "step and read one step late"},
            "e2e_verbatim_closure": {"value": vb_value, "unit": "it/s", "steps": vb_steps,
                                     "api": "same, with the verbatim denoising.ipynb c10 closure: EMA out_avg, 3 x PSNR on "
                                            "D2H copies of the 3x512x512 output, last_net = [x.detach().cpu() ...] of the 112 "
                                            "parameters every iteration"},
            "e2e_fast_verbatim_closure": {"value": fv_value, "unit": "it/s", "steps": fv_steps,
                                          "api": "utils.fast_closure.DenoisingClosure: the c10 logic (EMA, PSNR_noisy / PSNR_gt / "
                                                 "PSNR_gt_sm, back-tracking snapshot) with device-side PSNRs (dip_loss_mse) and a "
                                                 "device-side parameter snapshot; one 32-byte read-back per iteration"},
            "gpu_library_baseline": {"value": lib_value, "unit": "it/s", "n_gpus": 1,
                                     "what": "the same module tree executed by stock torch.cuda + cuDNN (cudnn.benchmark=True, "
                                             "TF32 convolutions = torch default), lean closure, torch.optim.Adam -- the "
                                             "reference's own GPU path on the same GPU (denoising.ipynb c3:17-19)",
                                     "speedup_value_per_gpu": (value / world) / lib_value if lib_value else None},
            "gpu_launches": int(launches_per_step * args.steps),
            "gpu_launches_per_step": int(launches_per_step),
            "roofline": roof,
            "roofline_dominant_launch": tensor_roof("tc_conv_kernel, level-0 3x3 conv 132->128 @512x512 fprop (largest launch)",
                                                    lambda r: r[0] == 0 and r[1] == big),
            "roofline_wgrad": tensor_roof("tc_wgrad_kernel (wgmma tf32, operands transposed in shared memory, split-K), all launches",
                                          lambda r: r[0] == 2),
            "roofline_hbm_all": hbm_roof("all HBM-bound launches of a step (sum of algorithmic bytes / sum of device time)",
                                         lambda r: r[0] >= 16, {"by_kernel": by_kernel}),
            "roofline_hbm": hbm_roof("k_bn_bwd_apply<plain>: BatchNorm+LeakyReLU backward (apply pass) behind the level-0 up "
                                     "conv, 128 ch @512x512 (largest HBM-bound launch)",
                                     lambda r: r[0] == 16 + 8 * 8 and r[1] == hbm_big,
                                     {"traffic": TRAFFIC.get("bn_bwd_apply_l0")}),
            "step_tflops": ALG_GFLOP_PER_ITER / 1000.0 / (step_ms / 1000.0),
            "config3_sr_x4_1024": sr_cfg,
            "per_rank": [{"psnr_gt_after_image": r[0], "final_loss": r[1], "it_per_s_image": r[2]} for r in recs],
        }
        if world == 1 and not args.no_cpu_baseline:
            # the reference arm on a bounded sample, in its own process (its `models` / `utils` are the reference's)
            env = dict(os.environ, DIP_REF_BUDGET_S="40")
            try:
                out = subprocess.run([sys.executable, os.path.abspath(__file__), "--impl", "reference", "--steps", "6",
                                      "--warmup", "2"], capture_output=True, text=True, env=env, timeout=900)
                ref_line = json.loads([ln for ln in out.stdout.splitlines() if ln.startswith("{")][-1])
                line["cpu_baseline"] = ref_line["cpu_baseline"]
            except Exception as e:   # the bench line must still come out
                line["cpu_baseline"] = {"value": None, "unit": "it/s", "cores": 0, "kind": "port", "sample": "failed: %r" % (e,)}
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


SR_ALG_GFLOP_PER_ITER = 1840.3   # the same network at 1024x1024 (4 x the 512x512 count), DESIGN.md section 3


def bench_sr_config(torch, de, models, peaks, dev, iters=100):
    """BASELINE.json configs[2] ("super-resolution x4 zebra 256->1024, skip net + Lanczos downsampler, bf16") on the runner:
    noise + forward + Lanczos-2 x4 operator + MSE on the 256^2 target + the operator's adjoint + backward + Adam per step.
    Timed in both tensor-core modes; the bf16 mode also gets a per-launch pass (CUDA events around every tensor-core launch
    of an eager step) for its roofline against the measured bf16 peak."""
    HS = WS = 1024
    gen = torch.Generator().manual_seed(7)
    z0 = (torch.rand(1, IN_CH, HS, WS, generator=gen) * 0.1).to(dev)
    target = torch.rand(1, OUT_CH, HS // 4, WS // 4, generator=gen).to(dev)
    down = models.Downsampler(n_planes=3, factor=4, kernel_type="lanczos2", phase=0.5, preserve_size=True)
    out = {"workload": "super-resolution x4: skip[128x5] in32 out3 bilinear at 1024x1024, Lanczos-2 operator to 256x256 in the loss, "
                       "noise+fwd+operator+MSE+adjoint+bwd+Adam per step (BASELINE.json configs[2]); synthetic target",
           "algorithmic_gflop_per_step": SR_ALG_GFLOP_PER_ITER}
    for prec_name, prec in (("tf32", de.PRECISION_TF32), ("bf16", de.PRECISION_BF16)):
        torch.manual_seed(0)
        net = models.get_net(IN_CH, "skip", "reflection", skip_n33d=128, skip_n33u=128, skip_n11=4, num_scales=5,
                             upsample_mode="bilinear").type(torch.cuda.FloatTensor)
        params = [p for p in net.parameters()]
        grads = [torch.zeros_like(p) for p in params]
        plan = de.Plan(IN_CH, OUT_CH, 5, 128, 4, True, HS, WS, precision=prec, device=dev)
        plan.bind(params, grads)
        for p_, g_ in zip(params, grads):
            p_.grad = g_
        opt = de.FusedAdam(params, lr=LR)
        opt._bind(grads)
        plan.set_downsampler(down.kernel, 4, down.pad)
        obuf = torch.empty(1, OUT_CH, HS, WS, device=dev)
        hist = torch.zeros(iters, dtype=torch.float64, device=dev)
        de.run_iterations(plan, opt, z0, target, None, 0.03, 99, 5, LR, out=obuf)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        de.run_iterations(plan, opt, z0, target, None, 0.03, 99, iters, LR, out=obuf, loss_hist=hist)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        rec = {"it_per_s": 1000.0 / ms, "ms_per_step": ms, "steps": iters, "step_tflops": SR_ALG_GFLOP_PER_ITER / ms,
               "loss_first": float(hist[0].item()), "loss_last": float(hist[-1].item())}
        # per-launch pass
        os.environ["DIP_NO_SIDE"] = "1"
        plan.set_timing(True)
        de.run_iterations(plan, opt, z0, target, None, 0.03, 99, 3, LR, out=obuf)
        torch.cuda.synchronize()
        records = plan.get_timing_records()
        plan.set_timing(False)
        os.environ.pop("DIP_NO_SIDE", None)
        peak = peaks["bf16_tflops"] * (1.0 if prec_name == "bf16" else 0.5)
        for nm, classes in (("conv_fprop_dgrad", (0, 1)), ("wgrad", (2,))):
            sel = [r for r in records if r[0] in classes]
            ms_, fl_ = sum(r[2] for r in sel), sum(r[1] for r in sel)
            ach = fl_ / (ms_ / 1000.0) / 1e12 if ms_ > 0 else 0.0
            rec["roofline_" + nm] = {"bound": "tensor", "achieved": ach, "peak": peak, "unit": "TFLOP/s", "frac": ach / peak,
                                     "launches_per_step": len(sel) // 3, "ms_per_step": ms_ / 3.0}
        fp = [r for r in records if r[0] == 0]
        big = max(fp, key=lambda r: r[1])
        rec["roofline_dominant_launch"] = {"kernel": "level-0 3x3 conv 132->128 @1024x1024 fprop", "bound": "tensor",
                                           "achieved": big[1] / (big[2] / 1000.0) / 1e12, "peak": peak, "unit": "TFLOP/s",
                                           "frac": big[1] / (big[2] / 1000.0) / 1e12 / peak}
        hb = [r for r in records if r[0] >= 16]
        ms_, by_ = sum(r[2] for r in hb), sum(r[1] for r in hb)
        rec["hbm_kernels"] = {"ms_per_step": ms_ / 3.0, "algorithmic_GB_per_s_fp32_bytes": by_ / (ms_ / 1000.0) / 1e9 if ms_ > 0 else 0.0}
        rec["peak_note"] = "peak = measured burst cuBLAS bf16 rate (MEASURED_PEAKS.json)" + ("" if prec_name == "bf16" else " / 2 (tf32)")
        del plan, opt
        # the same configuration end to end through the notebook-facing API (super-resolution.ipynb c10 without the logging):
        # net(net_input + noise) -> Downsampler -> MSELoss -> backward() -> optimize('adam', ...), loss read back every step
        from utils.common_utils import get_params
        from utils.common_utils import optimize as _opt
        import contextlib
        import io
        net.precision = prec_name
        for p_ in params:
            p_.grad = None
        dmod = down.type(torch.cuda.FloatTensor)
        mse = torch.nn.MSELoss().type(torch.cuda.FloatTensor)
        noise = z0.detach().clone()
        last = [0.0]

        def closure():
            out_hr = net(z0 + noise.normal_() * 0.03)
            total_loss = mse(dmod(out_hr), target)
            total_loss.backward()
            last[0] = total_loss.item()
            return total_loss

        def run(n):
            with contextlib.redirect_stdout(io.StringIO()):
                _opt("adam", get_params("net", net, z0), closure, LR, n)
        run(5)
        torch.cuda.synchronize()
        e0.record()
        run(50)
        e1.record()
        torch.cuda.synchronize()
        rec["e2e_it_per_s"] = 50.0 / (e0.elapsed_time(e1) / 1000.0)
        rec["e2e_api"] = "models.get_net(...).type(cuda) with net.precision = '%s', models.Downsampler, utils.optimize('adam', ...), loss.item() every step" % prec_name
        out[prec_name] = rec
        del net, params, grads, dmod
        torch.cuda.empty_cache()
    out["bf16_speedup"] = out["bf16"]["it_per_s"] / out["tf32"]["it_per_s"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the outputs of the last timed step as DIR/<name>.npy")
    args = ap.parse_args()
    if args.dump_outputs and args.impl != "ours":
        ap.error("--dump-outputs writes what the engine's timed steps computed; the reference arm has no such outputs")
    if args.impl == "reference":
        run_reference(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
