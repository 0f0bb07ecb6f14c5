"""Weight-gradient launches of the 512x512 flagship step (skip[128x5] in32 out3, skip channels 4, bilinear, tf32).

Prints, for every tc_wgrad_kernel launch of one step, its shape, its time (CUDA events around the launch, from
plan.get_timing_records(), class 2) and its rate, both algorithmic (2 * N * C * k^2 * pixels) and as executed (the
128 x n_cols accumulator tile over every pixel block of 32, padding included).  Then it times the graph-replayed runner in
two child processes, with and without DIP_DBG_SKIP_WGRAD=1 (no weight gradients at all): the difference is the most any
weight-gradient kernel can take off a step.

usage: python scripts/wgrad_shapes.py [--steps N]      (DIP_LIB selects another libdip.so build)
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H = W = 512
SCALES, CH, CS, IN_CH = 5, 128, 4, 32


def wgrad_cols(C):
    """accumulator columns per tap of the tensor-core weight gradient (ConvOp::wg_cols in engine.cu)"""
    return 136 if 128 < C <= 136 else (C + 31) // 32 * 32


def flagship_wgrads():
    """(name, C, k, out_h, out_w) of every tensor-core weight gradient of the flagship network"""
    convs = []
    for l in range(SCALES):
        Hl = H >> l
        cin = IN_CH if l == 0 else CH
        convs += [("L%d down1 3x3 s2" % l, cin, 3, Hl // 2, Hl // 2), ("L%d down2 3x3" % l, CH, 3, Hl // 2, Hl // 2),
                  ("L%d up 3x3" % l, CH + CS, 3, Hl, Hl), ("L%d 1x1" % l, CH, 1, Hl, Hl)]
    return convs


def child_records(steps):
    import torch
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "deep-image-prior_b200"))
    from oracle import dip_oracle as O
    import dip_engine as de
    cfg = O.SkipConfig(upsample_mode="bilinear", skip_channels=CS)
    params = [p.detach().cuda() for p in O.init_params(cfg, seed=0)]
    grads = [torch.zeros_like(p) for p in params]
    plan = de.Plan(IN_CH, 3, SCALES, CH, CS, True, H, W, precision=de.PRECISION_TF32)
    plan.bind(params, grads)
    adam = de.FusedAdam(params, lr=0.01)
    adam._bind(grads)
    z0 = torch.rand(1, IN_CH, H, W, device="cuda") * 0.1
    target = torch.rand(1, 3, H, W, device="cuda")
    out = torch.empty(1, 3, H, W, device="cuda")

    def run(n, hist=None):
        de.run_iterations(plan, adam, z0, target, None, 1 / 30., 1, n, 0.01, out=out, loss_hist=hist)

    run(10)
    torch.cuda.synchronize()
    if os.environ.get("WGRAD_SHAPES_MODE") == "time":
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run(steps)
        e1.record()
        torch.cuda.synchronize()
        print(json.dumps({"ms_per_step": e0.elapsed_time(e1) / steps}))
        return
    os.environ["DIP_NO_SIDE"] = "1"   # kernels timed one at a time
    plan.set_timing(True)
    run(steps)
    torch.cuda.synchronize()
    recs = plan.get_timing_records()
    plan.set_timing(False)
    print(json.dumps({"records": [list(r) for r in recs if r[0] == 2], "steps": steps}))


def child(mode, steps, extra_env=None):
    env = dict(os.environ, WGRAD_SHAPES_MODE=mode, **(extra_env or {}))
    out = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--steps", str(steps)], env=env,
                         capture_output=True, text=True, check=True)
    return json.loads([ln for ln in out.stdout.splitlines() if ln.startswith("{")][-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--child", action="store_true")
    args = ap.parse_args()
    if args.child:
        child_records(args.steps)
        return
    rec = child("records", args.steps)
    shapes = {}
    for name, C, k, oh, ow in flagship_wgrads():
        alg = 2.0 * CH * C * k * k * oh * ow
        exe = 2.0 * CH * wgrad_cols(C) * k * k * oh * ((ow + 31) // 32 * 32)
        shapes.setdefault(alg, []).append((name, exe))
    per = {}
    for _, fl, ms in rec["records"]:
        per.setdefault(fl, []).append(ms)
    print("%-32s %9s %8s %9s %9s" % ("wgrad launch", "GFLOP", "ms", "alg TF/s", "exec TF/s"))
    tot_ms = tot_alg = tot_exe = 0.0
    for fl in sorted(per, reverse=True):
        names = shapes.get(fl, [("(unknown shape)", fl)])
        ms = sum(per[fl]) / len(per[fl])          # every launch of this flop count, averaged over the steps
        per_step = len(per[fl]) / rec["steps"]   # launches of this flop count per step
        exe = names[0][1]
        label = " / ".join(n for n, _ in names)
        print("%-32s %9.2f %8.3f %9.1f %9.1f  x%g" % (label[:32], fl / 1e9, ms, fl / ms / 1e9, exe / ms / 1e9, per_step))
        tot_ms += ms * per_step
        tot_alg += fl * per_step
        tot_exe += exe * per_step
    print("all wgrad launches: %.3f ms/step, %.1f GFLOP/step algorithmic (%.1f TFLOP/s), %.1f executed (%.1f TFLOP/s)" %
          (tot_ms, tot_alg / 1e9, tot_alg / tot_ms / 1e9, tot_exe / 1e9, tot_exe / tot_ms / 1e9))
    steps = max(args.steps, 200)
    full = child("time", steps)["ms_per_step"]
    skip = child("time", steps, {"DIP_DBG_SKIP_WGRAD": "1"})["ms_per_step"]
    print("runner: %.3f ms/step (%.1f it/s); without weight gradients %.3f ms/step (%.1f it/s): at most %.1f%% of the step" %
          (full, 1000 / full, skip, 1000 / skip, 100 * (full - skip) / full))


if __name__ == "__main__":
    main()
