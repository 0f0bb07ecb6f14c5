"""Runner step time of the 512x512 denoising network (skip[128x5] in32 out3, skip channels 4, bilinear, reflection, tf32)
with each activation of models.skip's act_fun: 'LeakyReLU', 'Swish', 'ELU' and 'none'.

The four plans are built once in one process; the script then alternates them, `--rounds` times each, timing `--steps`
graph-replayed runner iterations per round with CUDA events after `--warmup` iterations of the same plan.  It prints one
JSON line with the card's name and power limit, the per-round ms/step of each kind, their medians and each median over
LeakyReLU's.

usage: python scripts/act_modes.py [--steps 200] [--warmup 20] [--rounds 5]      (DIP_LIB selects another libdip.so build)
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from pad_modes import CH, CS, H, IN_CH, SCALES, W, card  # noqa: E402

KINDS = ("LeakyReLU", "Swish", "ELU", "none")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "deep-image-prior_b200"))
    from oracle import dip_oracle as O
    import dip_engine as de
    if not torch.cuda.is_available():
        raise SystemExit("act_modes.py measures on the GPU; no CUDA device is visible")
    cfg = O.SkipConfig(upsample_mode="bilinear", skip_channels=CS)
    g = torch.Generator().manual_seed(0)
    z0 = (torch.rand(1, IN_CH, H, W, generator=g) * 0.1).cuda()
    target = torch.rand(1, 3, H, W, generator=g).cuda()
    runs = {}
    for act in KINDS:
        params = [p.detach().cuda().contiguous() for p in O.init_params(cfg, seed=0)]
        grads = [torch.zeros_like(p) for p in params]
        plan = de.Plan(IN_CH, 3, SCALES, CH, CS, True, H, W, precision=de.PRECISION_TF32, act=act)
        plan.bind(params, grads)
        for p, gb in zip(params, grads):
            p.grad = gb
        adam = de.FusedAdam(params, lr=0.01)
        adam._bind(grads)
        hist = torch.zeros(max(args.steps, args.warmup), dtype=torch.float64, device="cuda")
        runs[act] = (plan, adam, hist)
    ms = {act: [] for act in KINDS}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for act, (plan, adam, hist) in runs.items():
            de.run_iterations(plan, adam, z0, target, None, 1. / 30, 7, args.warmup, 0.01, loss_hist=hist)
            torch.cuda.synchronize()
            ev0.record()
            de.run_iterations(plan, adam, z0, target, None, 1. / 30, 7, args.steps, 0.01, loss_hist=hist)
            ev1.record()
            torch.cuda.synchronize()
            assert torch.isfinite(hist).all()
            ms[act].append(ev0.elapsed_time(ev1) / args.steps)
    med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
    print(json.dumps({"workload": "runner step, denoising 512x512 skip[128x5] cs4 bilinear reflection tf32", "card": card(),
                      "steps_per_round": args.steps, "warmup": args.warmup, "rounds": args.rounds,
                      "ms_per_step": ms, "median_ms_per_step": med,
                      "over_leaky_relu": {k: med[k] / med["LeakyReLU"] for k in KINDS}}))


if __name__ == "__main__":
    main()
