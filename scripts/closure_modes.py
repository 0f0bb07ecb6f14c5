"""What the denoising notebook's closure (denoising.ipynb c10: EMA out_avg, three PSNRs, back-tracking) costs in each of
the ways the project can run it, on the flagship network (skip, 128 wide, 4-channel skips, 5 scales, bilinear, tf32):

  lean      dip_run_iterations: noise -> forward -> MSE -> backward -> Adam, one CUDA graph per iteration (no closure)
  tracked   dip_run_iterations_tracked at c10's settings (exp_weight 0.99, show_every 100, 5 dB): the closure in the graph
  fast      utils.fast_closure.DenoisingClosure through utils.common_utils.optimize: one 32-byte read-back per iteration
  verbatim  the c10 closure as the notebook has it: three PSNRs through .cpu(), last_net through .cpu()

at 512 x 512 and 128 x 128.  Each mode has its own network (and plan, so no mode recaptures another's graph).  After a
warm-up, 5 rounds alternate the modes, each timing >= 200 iterations (50 for verbatim) between device synchronisations;
the medians are printed.  Before timing, the tracked runner at backtrack_db = 1e3 (snapshots saved, never restored) must
leave the same parameters as the lean runner from the same state, bit for bit.

    python scripts/closure_modes.py [--steps 200] [--rounds 5] [--json PATH]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "deep-image-prior_b200")]

import dip_engine as de                                         # noqa: E402
import models                                                   # noqa: E402
from utils.common_utils import get_noise, get_params, optimize  # noqa: E402
from utils.fast_closure import DenoisingClosure                 # noqa: E402

LR, SIGMA_REG, SEED = 0.01, 1. / 30, 1234
MODES = ["lean", "tracked", "fast", "verbatim"]


def make_net():
    torch.manual_seed(0)
    return models.get_net(32, "skip", "reflection", skip_n33d=128, skip_n33u=128, skip_n11=4, num_scales=5,
                          upsample_mode="bilinear").type(torch.cuda.FloatTensor)


def problem(n):
    g = torch.Generator().manual_seed(7)
    clean = torch.rand(1, 3, n, n, generator=g)
    noisy = (clean + torch.randn(1, 3, n, n, generator=g) * (25 / 255.)).clamp(0, 1)
    torch.manual_seed(1)
    z0 = get_noise(32, "noise", (n, n)).type(torch.cuda.FloatTensor).detach()
    return z0, clean.cuda(), noisy.cuda()


class Runner:
    """the device runner on a network of its own, with or without the tracker"""

    def __init__(self, z0, clean, noisy, tracked, backtrack_db=5.0):
        self.net = make_net()
        self.z0, self.noisy = z0, noisy
        self.plan, params = self.net._engine_state(z0)
        self.adam = de.FusedAdam(params, lr=LR)
        self.adam._bind(self.net._dip_grad_views)
        self.out = torch.empty(1, 3, z0.shape[2], z0.shape[3], device="cuda")
        self.tracker = de.Tracker(self.adam, tuple(self.out.shape), gt=clean, exp_weight=0.99, show_every=100,
                                  backtrack_db=backtrack_db) if tracked else None
        self.records = None

    def __call__(self, n):
        if self.tracker is not None and (self.records is None or self.records.shape[0] < n):
            self.records = torch.empty(n, de.RECORD, dtype=torch.float64, device="cuda")
        de.run_iterations(self.plan, self.adam, self.z0, self.noisy, None, SIGMA_REG, SEED, n, LR, out=self.out,
                          track=self.tracker, records=self.records)

    def params(self):
        return torch.cat([p.detach().reshape(-1) for p in self.net.parameters()])


def fast_mode(z0, clean, noisy):
    net = make_net()
    closure = DenoisingClosure(net, z0, noisy, clean, reg_noise_std=SIGMA_REG, exp_weight=0.99, show_every=100,
                               mse=torch.nn.MSELoss().type(torch.cuda.FloatTensor))
    return lambda n: optimize("adam", get_params("net", net, z0), closure, LR, n)


def verbatim_mode(z0, clean, noisy):
    net = make_net()
    mse = torch.nn.MSELoss().type(torch.cuda.FloatTensor)
    img_np, img_noisy_np = clean.cpu().numpy()[0], noisy.cpu().numpy()[0]
    noise = z0.detach().clone()
    st = {"i": 0, "out_avg": None, "last_net": None, "psrn_noisy_last": 0}

    def psnr_np(a, b):
        return 10 * np.log10(1.0 / np.mean((a.astype(np.float64) - b) ** 2))

    def closure():   # denoising.ipynb c10:8-56 without printing and plotting
        net_input = z0 + (noise.normal_() * SIGMA_REG)
        out = net(net_input)
        st["out_avg"] = out.detach() if st["out_avg"] is None else st["out_avg"] * 0.99 + out.detach() * (1 - 0.99)
        total_loss = mse(out, noisy)
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

    return lambda n: optimize("adam", get_params("net", net, z0), closure, LR, n)


def timed(fn, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn(n)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--verbatim-steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--sizes", default="512,128")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("closure_modes.py measures on the GPU; none is visible")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print("card: %s" % (card[torch.cuda.current_device()] if card else "unknown"))
    result = {"card": card[torch.cuda.current_device()] if card else None, "sizes": {}}
    for n in (int(x) for x in args.sizes.split(",")):
        z0, clean, noisy = problem(n)
        # parity: the tracker changes no training arithmetic when it restores nothing
        lean, ref = Runner(z0, clean, noisy, False), Runner(z0, clean, noisy, True, backtrack_db=1e3)
        lean(20)
        ref(20)
        torch.cuda.synchronize()
        assert (ref.records[:20, 5] != 2).all() and (ref.records[:20, 5] == 1).any()
        assert torch.equal(lean.params(), ref.params()), "tracked runner (no restore) != lean runner at %d^2" % n
        fns = {"lean": lean, "tracked": Runner(z0, clean, noisy, True), "fast": fast_mode(z0, clean, noisy),
               "verbatim": verbatim_mode(z0, clean, noisy)}
        steps = {m: args.verbatim_steps if m == "verbatim" else args.steps for m in MODES}
        for m in MODES:
            fns[m](5)   # warm-up: plans, graphs, allocator
        ms = {m: [] for m in MODES}
        for _ in range(args.rounds):
            for m in MODES:
                ms[m].append(timed(fns[m], steps[m]))
        med = {m: statistics.median(ms[m]) for m in MODES}
        result["sizes"][n] = {m: {"ms_per_iter": med[m], "it_per_s": 1e3 / med[m], "rounds_ms": ms[m],
                                  "steps": steps[m]} for m in MODES}
        print("%d x %d (median of %d rounds):" % (n, n, args.rounds))
        for m in MODES:
            print("  %-9s %8.3f ms/it  %8.1f it/s  x%.2f of lean   (rounds: %s)" % (
                m, med[m], 1e3 / med[m], med[m] / med["lean"], " ".join("%.3f" % x for x in ms[m])))
        del fns, lean, ref
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
