"""The envelope table (tests/envelope_cases.py) on the host: for every row, the unmodified reference's models.skip against
the oracle (parameters bit for bit, forward in fp64), the fp64 stage references composed stage by stage against the
oracle's autograd (output, every parameter gradient and dz), and models.skip's routing of the row to the engine.  These
hold the references that judge the engine in tests/test_envelope_gpu.py.  No GPU needed."""
import pytest
import torch

import models
from oracle import dip_oracle as O
from oracle import ref_harness
import envelope_cases as E
from test_stage_ref_cpu import check_composed

CASES = [(r.id, pad) for r in E.ROWS for pad in E.pads_of(r)]
IDS = ["%s_%s" % c for c in CASES]


@pytest.mark.skipif(not ref_harness.available(), reason="reference checkout not present")
@pytest.mark.parametrize("rid,pad", CASES, ids=IDS)
def test_reference_anchor(rid, pad):
    """the reference's network at the row's arguments: the oracle's init draws are its parameters bit for bit, and the
    oracle's forward is its forward in fp64"""
    row = E.BY_ID[rid]
    cfg = E.cfg_of(rid, pad)
    with ref_harness.reference_modules() as ref:
        torch.manual_seed(0)
        rnet = ref.models.skip(**E.skip_kwargs(row, pad))
        rparams = [p.detach().clone() for p in rnet.parameters()]
        rnet = rnet.double()
        z = torch.rand(1, row.in_ch, row.H, row.W, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
        rout = rnet(z).detach()
    params = O.init_params(cfg, seed=0)
    assert [tuple(p.shape) for p in rparams] == [tuple(p.shape) for p in params]
    for (name, _), a, b in zip(O.param_layout(cfg), rparams, params):
        assert torch.equal(a, b.detach()), name
    out = O.skip_forward([p.detach().double() for p in params], z, cfg).detach()
    assert out.shape == rout.shape and (out - rout).abs().max().item() <= 1e-12


@pytest.mark.parametrize("rid,pad", CASES, ids=IDS)
def test_composed_stages_reproduce_the_oracle(rid, pad):
    """tests/stage_ref.py composed stage by stage against the oracle's output and autograd gradients, dz included
    (tests/test_stage_ref_cpu.py's check)"""
    row = E.BY_ID[rid]
    check_composed(E.cfg_of(rid, pad), row.H, row.W, True)


@pytest.mark.parametrize("rid,pad", CASES, ids=IDS)
def test_models_skip_routes_the_row_to_the_engine(rid, pad):
    """models.skip at the row's arguments is accelerated, with the row's widths, skips, up-mode mask and padding, and its
    parameters are the oracle's init draws in the oracle's order"""
    row = E.BY_ID[rid]
    torch.manual_seed(0)
    net = models.skip(**E.skip_kwargs(row, pad))
    spec = net._dip_spec
    assert spec is not None and net._dip_why is None, net._dip_why
    L = row.L
    per = lambda x: list(x) if isinstance(x, (list, tuple)) else [x] * L   # noqa: E731
    assert spec["num_scales"] == L and spec["in_channels"] == row.in_ch and spec["out_channels"] == row.out_ch
    assert per(spec["channels"]) == row.down
    assert per(spec["channels"] if spec["channels_up"] is None else spec["channels_up"]) == row.up
    assert per(spec["skip_channels"]) == row.skips
    assert per(spec["bilinear"]) == [m == "bilinear" for m in row.modes]
    assert spec["pad"] == pad and spec["downsample_mode"] == row.downsample and spec["need_sigmoid"] == row.sigmoid
    cfg = E.cfg_of(rid, pad)
    for (name, shape), a, b in zip(O.param_layout(cfg), net.parameters(), O.init_params(cfg, seed=0)):
        assert tuple(a.shape) == tuple(shape) and torch.equal(a.detach(), b.detach()), name
    assert len(list(net.parameters())) == len(O.param_layout(cfg))
