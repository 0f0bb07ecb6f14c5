"""Verbatim-closure semantics at engine speed (SURVEY.md 8f.1) -- an OPT-IN helper, not part of the reference's surface.

The denoising notebook's closure (denoising.ipynb c10:8-56) does, every iteration, three device->host copies of the
3 x H x W output for skimage's compare_psnr, and `last_net = [x.detach().cpu() for x in net.parameters()]` -- 112 more
copies with a sync each.  None of that can be made cheap from below while the cell text stays as it is (the cost is in
`.cpu()` itself), so the unmodified notebook is bounded by those host round trips however fast the network is.  This module
keeps the SAME logic -- perturbed input, EMA `out_avg`, PSNR_noisy / PSNR_gt / PSNR_gt_sm, back-tracking to the last
good parameters when PSNR_noisy drops by more than 5 dB -- but keeps the quantities on the device:

  * PSNRs: the engine's fused MSE kernel (dip_loss_mse) on device tensors; nothing is copied;
  * parameter snapshot: one multi-tensor device copy into a second set of buffers (no host round trip);
  * per iteration exactly ONE 32-byte read-back [loss, PSNR_noisy, PSNR_gt, PSNR_gt_sm], which the back-tracking test
    needs on the host anyway.

    closure = DenoisingClosure(net, net_input, img_noisy_torch, img_torch, reg_noise_std=1. / 30, exp_weight=0.99)
    optimize('adam', get_params('net', net, net_input), closure, LR, num_iter)
    closure.history  ->  [(loss, psnr_noisy, psnr_gt, psnr_gt_sm), ...];  closure.out_avg  ->  the smoothed output

DenoisingRun keeps the same logic inside the device runner (dip_run_iterations_tracked): the EMA, the PSNRs, the
back-tracking decision and the parameter snapshot / restore are made on the device within each replayed step, so a run of
any length needs one read-back at its end instead of one per iteration:

    run = DenoisingRun(net, net_input, img_noisy_torch, img_torch, reg_noise_std=1. / 30, LR=0.01)
    run.run(num_iter)
    run.history  ->  [(loss, psnr_noisy, psnr_gt, psnr_gt_sm, action), ...];  run.out_avg, run.fallbacks, run.i
"""
import math

import torch


def mse_device(a, b):
    """mean((a - b)^2) as a 1-element float64 CUDA tensor, one launch of the engine's loss kernel, no sync."""
    import dip_engine as de
    a, b = a.detach().contiguous(), b.detach().contiguous()
    assert a.is_cuda and a.dtype == torch.float32 and a.shape == b.shape
    c = a.shape[1] if a.dim() == 4 else 1
    acc = torch.zeros(1, dtype=torch.float64, device=a.device)
    with torch.cuda.device(a.device):
        de.check(de.lib().dip_loss_mse(a.data_ptr(), b.data_ptr(), None, c, a.numel() // c, acc.data_ptr(), None,
                                       torch.cuda.current_stream().cuda_stream))
    return acc


def psnr_device(img_true, img_test):
    """skimage.measure.compare_psnr for float images in [0, 1] (data_range 1), on the device: 1-element CUDA tensor."""
    return -10.0 * torch.log10(mse_device(img_true, img_test))


class ParamSnapshot:
    """`last_net = [x.detach().cpu() ...]` / `net_param.data.copy_(new_param.cuda())` without leaving the device."""

    def __init__(self, params):
        self.params = list(params)
        self.saved = [torch.empty_like(p) for p in self.params]
        self.valid = False

    def save(self):
        torch._foreach_copy_(self.saved, [p.detach() for p in self.params])
        self.valid = True

    def restore(self):
        assert self.valid, "no snapshot taken yet"
        with torch.no_grad():
            torch._foreach_copy_([p.data for p in self.params], self.saved)


class DenoisingClosure:
    """denoising.ipynb c10 closure with device-side metrics (see the module docstring)."""

    def __init__(self, net, net_input, img_noisy_torch, img_torch=None, reg_noise_std=1. / 30, exp_weight=0.99,
                 show_every=100, mse=None, on_show=None):
        self.net, self.reg_noise_std, self.exp_weight, self.show_every = net, reg_noise_std, exp_weight, show_every
        self.net_input_saved = net_input.detach().clone()
        self.noise = net_input.detach().clone()
        self.img_noisy, self.img_gt = img_noisy_torch, img_torch
        self.mse = mse if mse is not None else torch.nn.MSELoss()
        self.on_show = on_show                 # optional callback(i, out, out_avg) every show_every iterations
        self.out_avg = None
        self.snapshot = ParamSnapshot(net.parameters())
        self.psrn_noisy_last = 0.0
        self.i = 0
        self.fallbacks = 0
        self.history = []
        self.net_input = net_input

    def __call__(self):
        if self.reg_noise_std > 0:
            self.net_input = self.net_input_saved + (self.noise.normal_() * self.reg_noise_std)
        out = self.net(self.net_input)
        od = out.detach()
        self.out_avg = od if self.out_avg is None else self.out_avg * self.exp_weight + od * (1 - self.exp_weight)
        total_loss = self.mse(out, self.img_noisy)
        total_loss.backward()
        gt = self.img_gt if self.img_gt is not None else self.img_noisy
        vals = torch.cat([total_loss.detach().double().reshape(1), psnr_device(self.img_noisy, od), psnr_device(gt, od),
                          psnr_device(gt, self.out_avg)]).cpu().tolist()             # the iteration's ONE read-back
        loss, psrn_noisy, psrn_gt, psrn_gt_sm = vals
        self.history.append((loss, psrn_noisy, psrn_gt, psrn_gt_sm))
        if self.on_show is not None and self.i % self.show_every == 0:
            self.on_show(self.i, od, self.out_avg)
        if self.i % self.show_every:                                                  # back-tracking, c10:41-52
            if psrn_noisy - self.psrn_noisy_last < -5 and self.snapshot.valid:
                self.fallbacks += 1
                self.snapshot.restore()
                return total_loss * 0
            self.snapshot.save()
            self.psrn_noisy_last = psrn_noisy
        self.i += 1
        return total_loss


class DenoisingRun:
    """The denoising.ipynb c10 closure in the device runner: noise -> forward -> MSE -> EMA, PSNRs, back-tracking ->
    backward -> Adam, one captured CUDA graph per iteration.  Same arguments as DenoisingClosure plus the Adam learning
    rate `LR` and the noise `seed` (Philox stream, offset = Adam step); `mse` may only be None or an nn.MSELoss, since the
    runner takes the MSE itself, and a host callback cannot run inside the device loop.  backtrack_db: the drop of
    psrn_noisy that restores the last good parameters (5 dB in c10:42).

    history rows: (loss, psnr_noisy, psnr_gt, psnr_gt_sm, action) with action 0 none, 1 saved, 2 restored.  Without
    img_torch the ground-truth PSNRs are taken against the noisy image, as DenoisingClosure does."""

    def __init__(self, net, net_input, img_noisy_torch, img_torch=None, reg_noise_std=1. / 30, exp_weight=0.99,
                 show_every=100, mse=None, on_show=None, LR=0.01, seed=0, backtrack_db=5.0):
        import dip_engine as de
        if mse is not None and type(mse) is not torch.nn.MSELoss:
            raise ValueError("dip-b200: DenoisingRun takes the loss as the runner's MSE; mse must be None or nn.MSELoss()")
        if on_show is not None:
            raise ValueError("dip-b200: DenoisingRun cannot call on_show from inside the device loop; "
                             "read out_avg between run() calls")
        if getattr(net, "_dip_spec", None) is None:
            raise ValueError("dip-b200: DenoisingRun needs a network that runs on the engine (%s)"
                             % getattr(net, "_dip_why", "not a models.skip network"))
        if net_input.requires_grad:
            raise ValueError("dip-b200: DenoisingRun does not optimise the network input (OPT_OVER 'net,input')")
        self.z = net_input.detach().contiguous()
        self.plan, params = net._engine_state(self.z)
        if self.plan.desc.input_grad:
            raise ValueError("dip-b200: DenoisingRun does not run plans with input_grad")
        self.net, self.LR, self.seed, self.reg_noise_std = net, float(LR), int(seed), float(reg_noise_std)
        self.target = img_noisy_torch.detach().to(self.z.device, torch.float32).contiguous()
        gt = img_torch if img_torch is not None else img_noisy_torch
        self.adam = de.FusedAdam(params, lr=self.LR)
        self.adam._bind(net._dip_grad_views)
        self.out = torch.empty((1, self.plan.desc.out_channels, self.plan.H, self.plan.W), dtype=torch.float32,
                               device=self.z.device)
        self.tracker = de.Tracker(self.adam, tuple(self.out.shape), gt=gt, exp_weight=exp_weight, show_every=show_every,
                                  backtrack_db=backtrack_db)
        self.i = 0
        self.fallbacks = 0
        self.history = []

    @property
    def out_avg(self):
        return self.tracker.out_avg

    def run(self, num_iter):
        """num_iter iterations in one runner call, then one read-back of their records"""
        import dip_engine as de
        if num_iter <= 0:
            return self.history
        records = torch.empty((num_iter, de.RECORD), dtype=torch.float64, device=self.z.device)
        de.run_iterations(self.plan, self.adam, self.z, self.target, None, self.reg_noise_std, self.seed, num_iter, self.LR,
                          out=self.out, track=self.tracker, records=records)
        rows = records.cpu().tolist()
        for loss, psnr_noisy, psnr_gt, psnr_gt_sm, i, action in rows:
            self.history.append((loss, psnr_noisy, psnr_gt, psnr_gt_sm, int(action)))
            self.fallbacks += int(action) == de.ACTION_RESTORED
        last = rows[-1]
        self.i = int(last[4]) + (int(last[5]) != de.ACTION_RESTORED)
        return self.history
