"""The device runner with the denoising closure's tracker (dip_run_iterations_tracked: EMA out_avg, three PSNRs and the
back-tracking of denoising.ipynb c10:8-52 inside the captured step), against torch and fp64 at the engine's own buffers
(H100).

Configurations are test_runner_steps_gpu's runner configurations (plan, FusedAdam at lr = 0.01, sigma = 1/30), each with
a clean image gt ~ U(0, 1) at the output's size (the high-resolution size for super-resolution).  With show_every = 3 a
run of one-iteration calls goes through every branch of the rule in a known order:

    backtrack_db   iterations   actions (i before)
    -1e3           4            none (0), save (1), restore (2), restore (2)      every eligible iteration drops
    +1e3           3            save (2), none (3), save (4)                      none does
    5              2            the c10 rule on the engine's own PSNRs

After each call, from the buffers the engine left (teacher forcing):

* EMA: out_avg is bit for bit `prev * w + out * (1 - w)` evaluated by torch on the GPU (after the first call: `out`);
* PSNRs: psnr_target = -10 log10(loss record) to fp64 rounding, the loss record is the loss slot bit for bit; psnr_gt and
  psnr_gt_sm are within (10 / ln 10) r / (1 - r) of the fp64 PSNRs of the engine's out / out_avg against gt, where
  r = (gamma_{k+13} L + blocks 2^-49) / L is k_mse's relative bound (test_runner_steps_gpu's loss-slot bound, D = 0);
* rule: the recorded i and action, and the state, equal a Python replay of c10:41-52 over the recorded psnr_target;
* save: the snapshot is the parameters the forward used, bit for bit, and p', m', v' are within the Adam bounds of
  test_runner_steps_gpu from them;  restore: the snapshot is unchanged and p', m', v' are within the Adam bounds of
  Adam(snapshot, g, m, v).
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import test_runner_steps_gpu as RS

pytestmark = pytest.mark.gpu
LR, SIGMA, SEED, BETAS, EPS, U = RS.LR, RS.SIGMA, RS.SEED, RS.BETAS, RS.EPS, RS.U
EXP_WEIGHT = 0.99
SHOW_EVERY = 3
# (backtrack_db, one-iteration calls)
SCHEDULE = [(-1e3, 4), (1e3, 3), (5.0, 2)]
TRACK_CONFIGS = ["denoise_cs4_tf32", "denoise_cs4_bf16", "denoise_cs4_fp32", "inpaint_cs128_tf32", "sr_cs4_bf16"]
PSNR = {}   # cid -> worst |psnr error| / bound


def replay(state, psnr, show_every, db):
    """c10:41-52 (DenoisingClosure's restatement) on (i, psnr_last, has_snapshot, fallbacks) -> (action, new state)"""
    i, last, has, fb = state
    if show_every > 0 and i % show_every:
        if psnr - last < -db and has:
            return 2, (i, last, has, fb + 1)
        return 1, (i + 1, psnr, True, fb)
    return 0, (i + 1, last, has, fb)


def read_state(tracker):
    s = tracker.state.cpu()
    last = s[:8].view(torch.float64).item()
    i, action, has_avg, has_snap, fallbacks, _ = s[8:].view(torch.int32).tolist()
    return dict(i=i, action=action, has_avg=has_avg, has_snapshot=has_snap, fallbacks=fallbacks, psnr_last=last)


def psnr_bound(n, L):
    blocks = min(-(-n // 256), RS.MSE_BLOCK_CAP)
    k = -(-n // (256 * blocks))
    r = (RS.gamma(k + 13) * L + blocks * 2.0 ** -49) / L
    return 10.0 / math.log(10.0) * r / (1 - r) + 1e-12


class TrackRunner(RS.Runner):
    """a runner configuration with a Tracker of its FusedAdam"""

    def __init__(self, cid, with_gt=True, **kw):
        import dip_engine as de
        super().__init__(cid)
        g = torch.Generator().manual_seed(11)
        self.gt = torch.rand(tuple(self.out.shape), generator=g).cuda() if with_gt else None
        self.tracker = de.Tracker(self.adam, tuple(self.out.shape), gt=self.gt, **kw)

    def run(self, iters, **kw):
        import dip_engine as de
        records = torch.full((iters, de.RECORD), -7.0, dtype=torch.float64, device="cuda")
        hist = torch.full((iters,), -1.0, dtype=torch.float64, device="cuda")
        de.run_iterations(self.plan, self.adam, self.z0, self.target, self.mask, SIGMA, SEED, iters, LR, out=self.out,
                          loss_hist=hist, track=self.tracker, records=records, **kw)
        torch.cuda.synchronize()
        return records, hist


def check_psnr(tag, cid, got, img, gt):
    d = img.double() - gt.double()
    L = (d * d).mean().item()
    ref = -10.0 * math.log10(L)
    tol = psnr_bound(img.numel(), L)
    PSNR[cid] = max(PSNR.get(cid, 0.0), abs(got - ref) / tol)
    assert abs(got - ref) <= tol, "[%s] PSNR %.17g, fp64 %.17g, bound %.3g" % (tag, got, ref, tol)


@pytest.mark.parametrize("cid", TRACK_CONFIGS)
def test_tracked_calls_step_by_step(cid):
    r = TrackRunner(cid, exp_weight=EXP_WEIGHT, show_every=SHOW_EVERY)
    tr, adam = r.tracker, r.adam
    state = (0, 0.0, False, 0)
    expect = [0, 1, 2, 2, 1, 0, 1]   # the actions the first two phases force
    n = 0
    for db, calls in SCHEDULE:
        tr.backtrack_db = db
        for _ in range(calls):
            tag = "%s call %d (backtrack_db %g)" % (cid, n, db)
            step0 = adam.step_count
            prev_avg = tr.out_avg.clone()
            snap0 = tr.snapshot.clone()
            before = (RS.flat(r.params).clone(), adam.m_flat.clone(), adam.v_flat.clone())
            rec, hist = r.run(1)
            row = rec[0].tolist()
            out = r.out
            # EMA
            want = out.clone() if n == 0 else prev_avg * EXP_WEIGHT + out * (1 - EXP_WEIGHT)
            assert torch.equal(tr.out_avg, want), "[%s] out_avg != torch's EMA: max |diff| %.3g" % (
                tag, (tr.out_avg - want).abs().max().item())
            # PSNRs
            assert row[0] == hist[0].item(), "[%s] loss record %r, loss slot %r" % (tag, row[0], hist[0].item())
            want_t = (-10.0 * torch.log10(hist[:1])).item()
            assert math.isclose(row[1], want_t, rel_tol=1e-15), "[%s] psnr_target %r, -10 log10(loss) %r" % (tag, row[1], want_t)
            check_psnr(tag + " psnr_gt", cid, row[2], out, r.gt)
            check_psnr(tag + " psnr_gt_sm", cid, row[3], tr.out_avg, r.gt)
            # rule
            action, state = replay(state, row[1], SHOW_EVERY, db)
            if n < len(expect):
                assert action == expect[n], "[%s] the schedule should force action %d, the replay gives %d" % (tag, expect[n], action)
            assert (row[4], row[5]) == (state[0] - (action != 2), action), \
                "[%s] record i %r action %r, replay: action %d, state %s" % (tag, row[4], row[5], action, state)
            st = read_state(tr)
            assert (st["i"], st["action"], st["has_avg"], st["has_snapshot"], st["fallbacks"]) == (
                state[0], action, 1, int(state[2]), state[3]), "[%s] state %s, replay %s" % (tag, st, state)
            assert st["psnr_last"] == state[1], "[%s] psnr_last %r, replay %r" % (tag, st["psnr_last"], state[1])
            # Adam with the action
            after = (RS.flat(r.params), adam.m_flat, adam.v_flat)
            g = RS.flat(r.grads)
            if action == 2:
                assert torch.equal(tr.snapshot, snap0), "[%s] a restore changed the snapshot" % tag
                RS.check_adam("tracked restore", (snap0, before[1], before[2]), g, after, LR, BETAS, EPS, step0 + 1)
            else:
                if action == 1:
                    assert torch.equal(tr.snapshot, before[0]), "[%s] the snapshot is not the forward's parameters" % tag
                else:
                    assert torch.equal(tr.snapshot, snap0), "[%s] the snapshot changed without a save" % tag
                RS.check_adam("tracked", before, g, after, LR, BETAS, EPS, step0 + 1)
            n += 1
    print("[runner track] %s: worst PSNR |err|/bound %.3g; ADAM %s" % (cid, PSNR.get(cid, 0.0), RS.ADAM))


def test_tracked_without_gt_gives_nan_psnrs():
    r = TrackRunner("denoise_cs4_fp32", with_gt=False, show_every=SHOW_EVERY)
    rec, hist = r.run(3)
    rec = rec.cpu()
    assert torch.isnan(rec[:, 2:4]).all(), rec
    assert torch.isfinite(rec[:, [0, 1, 4, 5]]).all(), rec
    assert torch.equal(rec[:, 0], hist.cpu())


def test_tracked_training_unchanged():
    """at backtrack_db = 1e3 nothing is restored: loss, out, p, m, v equal the untracked runner's bit for bit"""
    import dip_engine as de
    a = RS.Runner("denoise_cs4_tf32")
    b = TrackRunner("denoise_cs4_tf32", show_every=SHOW_EVERY, backtrack_db=1e3)
    assert torch.equal(RS.flat(a.params), RS.flat(b.params))
    ha = torch.zeros(5, dtype=torch.float64, device="cuda")
    de.run_iterations(a.plan, a.adam, a.z0, a.target, a.mask, SIGMA, SEED, 5, LR, out=a.out, loss_hist=ha)
    rec, hb = b.run(5)
    assert (rec[:, 5] != 2).all()
    for name, x, y in (("loss", ha, hb), ("out", a.out, b.out), ("p", RS.flat(a.params), RS.flat(b.params)),
                       ("m", a.adam.m_flat, b.adam.m_flat), ("v", a.adam.v_flat, b.adam.v_flat)):
        assert torch.equal(x, y), "%s differs: max |diff| %.3g" % (name, (x - y).abs().max().item())


def test_tracked_chunked_calls_and_eager_loop():
    """3 + 4 iterations equal 7 in one call (records, out_avg, snapshot, state), and DIP_NO_GRAPH=1 gives the same records"""
    kw = dict(show_every=SHOW_EVERY, backtrack_db=5.0)
    a = TrackRunner("denoise_cs4_tf32", **kw)
    ra = torch.cat([a.run(3)[0], a.run(4)[0]])
    b = TrackRunner("denoise_cs4_tf32", **kw)
    rb = b.run(7)[0]
    assert torch.equal(ra, rb), (ra, rb)
    for name in ("out_avg", "snapshot", "state"):
        assert torch.equal(getattr(a.tracker, name), getattr(b.tracker, name)), name
    assert torch.equal(RS.flat(a.params), RS.flat(b.params))
    with RS.environment(DIP_NO_GRAPH="1"):
        c = TrackRunner("denoise_cs4_tf32", **kw)
        rc = c.run(7)[0]
    assert torch.equal(rb, rc), (rb, rc)
    assert torch.equal(b.tracker.out_avg, c.tracker.out_avg) and torch.equal(b.tracker.state, c.tracker.state)


def test_tracked_refuses_invalid_fields_before_launching():
    import dip_engine as de
    r = TrackRunner("denoise_cs4_fp32", show_every=SHOW_EVERY)
    records = torch.full((2, de.RECORD), -7.0, dtype=torch.float64, device="cuda")
    p0, out0 = RS.flat(r.params).clone(), r.out.clone()
    torch.cuda.synchronize()
    for field, value, word in [("exp_weight", 1.0, "exp_weight"), ("exp_weight", -0.5, "exp_weight"),
                               ("exp_weight", float("nan"), "exp_weight"), ("show_every", -1, "show_every"),
                               ("backtrack_db", float("nan"), "backtrack_db"), ("out_avg", None, "out_avg"),
                               ("snapshot", None, "snapshot"), ("state", None, "state"), ("records", None, "records")]:
        t = r.tracker.struct(records)
        setattr(t, field, value)
        rc = de.lib().dip_run_iterations_tracked(r.plan.h, r.adam.h, de._ptr(r.z0), de._ptr(r.target), None, SIGMA, SEED,
                                                 0, 2, LR, de._ptr(r.out), None, ctypes.byref(t), de._stream())
        err = de.lib().dip_last_error().decode()
        assert rc != 0 and word in err, (field, value, rc, err)
    torch.cuda.synchronize()
    assert (records == -7.0).all() and torch.equal(RS.flat(r.params), p0) and torch.equal(r.out, out0)
    assert (r.tracker.state == 0).all() and (r.tracker.out_avg == 0).all()
    with pytest.raises(ValueError, match="records"):
        de.run_iterations(r.plan, r.adam, r.z0, r.target, None, SIGMA, SEED, 2, LR, track=r.tracker)


# ------------------------------------------------------------------------------------------------ DenoisingRun
def f16_crop(n=128):
    from PIL import Image
    from utils.common_utils import pil_to_np
    from utils.denoising_utils import get_noisy_image
    import os
    img = Image.open(os.path.join(os.path.dirname(__file__), "golden", "data", "F16_GT.png"))
    img = img.crop((0, 0, n, n))
    img_np = pil_to_np(img)
    np.random.seed(0)
    _, noisy_np = get_noisy_image(img_np, 25 / 255.)
    return torch.from_numpy(img_np)[None].float().cuda(), torch.from_numpy(noisy_np)[None].float().cuda()


def make_net(kind, seed):
    import models
    from utils.common_utils import get_noise
    torch.manual_seed(seed)
    if kind == "snail":   # denoising.ipynb c8:17-23
        net = models.skip(3, 3, num_channels_down=[8, 16, 32, 64, 128], num_channels_up=[8, 16, 32, 64, 128],
                          num_channels_skip=[0, 0, 0, 4, 4], upsample_mode="bilinear", need_sigmoid=True, need_bias=True,
                          pad="reflection", act_fun="LeakyReLU")
        depth = 3
    else:                 # c8's F16 network
        net = models.get_net(32, "skip", "reflection", skip_n33d=128, skip_n33u=128, skip_n11=4, num_scales=5,
                             upsample_mode="bilinear")
        depth = 32
    net = net.type(torch.cuda.FloatTensor)
    torch.manual_seed(seed + 1)
    z = get_noise(depth, "noise", (128, 128)).type(torch.cuda.FloatTensor).detach()
    return net, z


@pytest.mark.parametrize("kind", ["snail", "f16"])
def test_denoising_run(kind):
    import dip_engine as de
    from utils.fast_closure import DenoisingRun
    gt, noisy = f16_crop()
    kw = dict(reg_noise_std=1. / 30, exp_weight=0.99, show_every=SHOW_EVERY, LR=0.01, seed=3)
    net1, z1 = make_net(kind, 0)
    one = DenoisingRun(net1, z1, noisy, gt, **kw)
    one.run(10)
    net2, z2 = make_net(kind, 0)
    two = DenoisingRun(net2, z2, noisy, gt, **kw)
    two.run(5)
    two.run(5)
    assert one.history == two.history
    assert torch.equal(one.out_avg, two.out_avg)
    assert torch.equal(RS.flat(list(net1.parameters())), RS.flat(list(net2.parameters())))
    assert (one.i, one.fallbacks) == (two.i, two.fallbacks)
    # the history is the engine's records: the same state driven through run_iterations + Tracker directly
    net3, z3 = make_net(kind, 0)
    plan, params = net3._engine_state(z3)
    adam = de.FusedAdam(params, lr=0.01)
    adam._bind(net3._dip_grad_views)
    out = torch.empty(1, 3, 128, 128, device="cuda")
    tracker = de.Tracker(adam, tuple(out.shape), gt=gt, exp_weight=0.99, show_every=SHOW_EVERY)
    records = torch.empty(10, de.RECORD, dtype=torch.float64, device="cuda")
    de.run_iterations(plan, adam, z3, noisy, None, 1. / 30, 3, 10, 0.01, out=out, track=tracker, records=records)
    rows = [tuple(r[:4]) + (int(r[5]),) for r in records.cpu().tolist()]
    assert rows == one.history
    assert tracker.i == one.i and tracker.fallbacks == one.fallbacks
    # the rule over the recorded PSNRs, and fallbacks from the actions
    state = (0, 0.0, False, 0)
    for row in one.history:
        action, state = replay(state, row[1], SHOW_EVERY, 5.0)
        assert action == row[4]
    assert state[0] == one.i and state[3] == one.fallbacks == sum(r[4] == 2 for r in one.history)
    assert all(torch.isfinite(p).all() for p in net1.parameters())
    # every eligible iteration restores once a snapshot exists
    net4, z4 = make_net(kind, 0)
    forced = DenoisingRun(net4, z4, noisy, gt, backtrack_db=-1e3, **kw)
    forced.run(6)
    assert [r[4] for r in forced.history] == [0, 1, 2, 2, 2, 2]
    assert forced.fallbacks == 4 and forced.i == 2
    assert all(torch.isfinite(p).all() for p in net4.parameters())


def test_denoising_run_refuses_what_it_cannot_run():
    from utils.fast_closure import DenoisingRun
    gt, noisy = f16_crop()
    net, z = make_net("snail", 0)
    with pytest.raises(ValueError, match="on_show"):
        DenoisingRun(net, z, noisy, gt, on_show=lambda *a: None)
    with pytest.raises(ValueError, match="input"):
        DenoisingRun(net, z.clone().requires_grad_(True), noisy, gt)
    with pytest.raises(ValueError, match="MSELoss"):
        DenoisingRun(net, z, noisy, gt, mse=torch.nn.L1Loss())
    import models
    off = models.skip(3, 3, filter_size_down=5).type(torch.cuda.FloatTensor)   # not a configuration of the engine
    with pytest.raises(ValueError, match="engine"):
        DenoisingRun(off, z, noisy, gt)
