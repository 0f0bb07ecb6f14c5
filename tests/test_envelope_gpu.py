"""The envelope table (tests/envelope_cases.py) on the engine (H100): 1 to 8 scales, every width class, unequal down / up
widths, input depths 1 to 100, 1 to 4 outputs.  Every stage of one forward + backward is checked against its fp64
reference at the engine's own inputs, in fp32, tf32 and bf16, with every registered buffer NaN-filled first (the
machinery and tolerances of tests/test_stages_gpu.py, unchanged); rows marked zero_pad run again with pad='zero' and
exact-zero halos.  The device runner runs at lr = 0 on three rows (the split-noise path at W % 4 = 2, masked inpainting,
x4 super-resolution), and three rows go through models.skip against the oracle's fp64 autograd."""
import torch
import torch.nn.functional as F
import pytest

from oracle import dip_oracle as O
import envelope_cases as E
import test_stages_gpu as TS

pytestmark = pytest.mark.gpu
MODES = ["fp32", "tf32", "bf16"]
STAGE_CASES = [(r.id, pad) for r in E.ROWS for pad in E.pads_of(r)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("rid,pad", STAGE_CASES, ids=["%s_%s" % c for c in STAGE_CASES])
def test_every_stage_envelope(rid, pad, mode):
    row = E.BY_ID[rid]
    TS.run_direct(E.cfg_of(rid, pad), row.H, row.W, mode, row.input_grad)
    TS.print_table()


@pytest.mark.parametrize("task,rid,H,W,mode", [("denoise", "L1", 10, 14, "tf32"), ("denoise", "L1", 10, 14, "bf16"),
                                                ("inpaint", "L4", 32, 48, "tf32"), ("sr", "rev5", 128, 128, "bf16")])
def test_every_stage_envelope_runner(task, rid, H, W, mode):
    TS.run_runner(E.cfg_of(rid), H, W, mode, task)
    TS.print_table()


@pytest.mark.parametrize("rid", [r.id for r in E.ROWS if r.module])
def test_models_skip_vs_oracle_fp32(rid):
    """models.skip(...) at the row's arguments, precision 'fp32', one forward + backward with dL/d(input): the spec ->
    Plan mapping, against the oracle's fp64 autograd at the bounds of test_variants.py's
    test_input_gradient_and_no_sigmoid_vs_oracle"""
    import models
    row = E.BY_ID[rid]
    cfg = E.cfg_of(rid)
    params = O.init_params(cfg, seed=0, dtype=torch.float64)
    gen = torch.Generator().manual_seed(2)
    z0 = (torch.rand(1, row.in_ch, row.H, row.W, generator=gen, dtype=torch.float64) * 0.1).requires_grad_(True)
    target = torch.rand(1, row.out_ch, row.H, row.W, generator=gen, dtype=torch.float64)
    out_ref = O.skip_forward(params, z0, cfg)
    grads_ref = torch.autograd.grad(O.mse_loss(out_ref, target), [z0] + params)

    torch.manual_seed(0)
    net = models.skip(**E.skip_kwargs(row)).type(torch.cuda.FloatTensor)
    assert net._dip_spec is not None, net._dip_why
    net.precision = "fp32"
    zd = z0.detach().float().cuda().requires_grad_(True)
    out = net(zd)
    F.mse_loss(out, target.float().cuda()).backward()
    err = (out.detach().double().cpu() - out_ref.detach()).abs().max().item()
    assert err < 5e-4, err

    def rel(a, b):
        a = a.double().cpu()
        return ((a - b).norm() / (b.norm() + 1e-30)).item()
    assert zd.grad is not None and rel(zd.grad, grads_ref[0]) < 3e-2, rel(zd.grad, grads_ref[0])
    gmax = max(g.norm().item() for g in grads_ref[1:])
    names = [n for n, _ in O.param_layout(cfg)]
    for name, p, g in zip(names, net.parameters(), grads_ref[1:]):
        if g.norm().item() > 1e-4 * gmax:
            assert rel(p.grad, g) < 3e-2, (name, rel(p.grad, g))
