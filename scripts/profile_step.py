"""Runs N iterations of the device runner (a workload to profile, e.g. with torch.profiler). usage: profile_step.py [iters] [H] [W]
env: DIP_PROF_CS=4|128 (skip channels), DIP_PROF_MODE=bilinear|nearest, DIP_PROF_SR=1 (x4 Lanczos-2 downsampler in the loss),
DIP_PROF_MASK=1 (masked MSE), DIP_PROF_PREC=tf32|fp32|bf16"""
import os, sys, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "deep-image-prior_b200"))
from oracle import dip_oracle as O
import dip_engine as de
iters = int(sys.argv[1]) if len(sys.argv) > 1 else 3
H = int(sys.argv[2]) if len(sys.argv) > 2 else 512
W = int(sys.argv[3]) if len(sys.argv) > 3 else 512
CS = int(os.environ.get("DIP_PROF_CS", "4"))
MODE = os.environ.get("DIP_PROF_MODE", "bilinear")
SR = os.environ.get("DIP_PROF_SR") is not None
cfg = O.SkipConfig(upsample_mode=MODE, skip_channels=CS)
params = [p.detach().cuda() for p in O.init_params(cfg, seed=0)]
grads = [torch.zeros_like(p) for p in params]
PREC = os.environ.get("DIP_PROF_PREC", "tf32")
plan = de.Plan(32, 3, 5, 128, CS, MODE == "bilinear", H, W,
               precision={"tf32": de.PRECISION_TF32, "fp32": de.PRECISION_FP32, "bf16": de.PRECISION_BF16}[PREC])
plan.bind(params, grads)
for p, g in zip(params, grads):
    p.grad = g
adam = de.FusedAdam(params, lr=0.01)
adam._bind(grads)
z0 = torch.rand(1, 32, H, W, device="cuda") * 0.1
target = torch.rand(1, 3, H // 4, W // 4, device="cuda") if SR else torch.rand(1, 3, H, W, device="cuda")
if SR:
    plan.set_downsampler(O.down_kernel(4, "lanczos2", 0.5), 4, 6)
mask = None
if os.environ.get("DIP_PROF_MASK") is not None:
    mask = (torch.rand(1, 1, target.shape[2], target.shape[3], device="cuda") > 0.05).float()
out = torch.empty(1, 3, H, W, device="cuda")
hist = torch.zeros(iters, dtype=torch.float64, device="cuda")
if os.environ.get("DIP_PROF_TIME") is not None:   # plain timing of the graph-replayed runner (it/s), no profiler
    de.run_iterations(plan, adam, z0, target, mask, 1 / 30., 1, 5, 0.01, out=out)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    de.run_iterations(plan, adam, z0, target, mask, 1 / 30., 1, iters, 0.01, out=out, loss_hist=hist)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    print("config %s cs=%d mode=%s sr=%s mask=%s %dx%d: %.3f ms/iter = %.1f it/s; loss first %.5f last %.5f" % (
        PREC, CS, MODE, SR, mask is not None, H, W, ms, 1000.0 / ms, hist[0].item(), hist[-1].item()))
else:
    de.run_iterations(plan, adam, z0, target, mask, 1 / 30., 1, iters, 0.01, out=out, loss_hist=hist)
    torch.cuda.synchronize()
print("done", plan.num_launches())
