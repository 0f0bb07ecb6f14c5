"""dip_plan_num_launches against what the plan really enqueues: one plan.forward and one plan.backward, each captured
into a CUDA graph of its own (eager launches, no side streams), must hold exactly as many nodes (kernel launches,
memsets, copies) as the plan reports for that pass.  bench.py reports this count as launches_per_step."""
import ctypes

import pytest
import torch

from oracle import dip_oracle as O
import envelope_cases as E
from test_stages_gpu import make_plan, params_for

pytestmark = pytest.mark.gpu

# (network, H, W, precision mode, pad, input_grad, x4 downsampler set as for the runner's super-resolution task)
CASES = [("cs4", 64, 96, "tf32", "reflection", False, False), ("cs128", 96, 64, "tf32", "reflection", False, False),
         ("kate", 96, 64, "fp32", "reflection", False, False), ("kate", 96, 64, "bf16", "reflection", False, False),
         ("snail", 64, 96, "bf16", "reflection", False, False), ("ingrad", 64, 96, "fp32", "zero", True, False),
         ("cs4", 256, 256, "bf16", "reflection", False, True)]


def cudart():
    """the CUDA runtime library torch has loaded (other packages may bring copies under other names)"""
    name = "libcudart.so." + torch.version.cuda.split(".")[0]
    with open("/proc/self/maps") as f:
        paths = {line.split()[-1] for line in f if line.rstrip().endswith("/" + name)}
    assert len(paths) == 1, paths
    lib = ctypes.CDLL(paths.pop())
    lib.cudaGraphGetNodes.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(ctypes.c_size_t)]
    return lib


def graph_nodes(fn):
    g = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(g):
        fn()
    n = ctypes.c_size_t(0)
    assert cudart().cudaGraphGetNodes(ctypes.c_void_p(g.raw_cuda_graph()), None, ctypes.byref(n)) == 0
    return n.value


@pytest.mark.parametrize("case", CASES, ids=["%s_%dx%d_%s_%s%s%s" % (c[0], c[1], c[2], c[3], c[4], "_ingrad" * c[5], "_down" * c[6])
                                             for c in CASES])
def test_num_launches_equals_graph_nodes(case, monkeypatch):
    kind, H, W, mode, pad, input_grad, down = case
    monkeypatch.setenv("DIP_NO_GRAPH", "1")
    monkeypatch.setenv("DIP_NO_SIDE", "1")
    cfg = E.cfg_of(kind, pad=pad)
    plan = make_plan(cfg, H, W, mode, input_grad)
    if down:
        kern = O.down_kernel(4, "lanczos2", 0.5)
        plan.set_downsampler(torch.from_numpy(kern).float(), 4, O.down_pad(kern.shape[0], 4))
    params = [p.cuda().contiguous() for p in params_for(cfg)]
    plan.bind(params, [torch.zeros_like(p) for p in params])
    z = torch.rand(1, cfg.in_channels, H, W, device="cuda")
    out = torch.empty(1, cfg.out_channels, H, W, device="cuda")
    dout = torch.rand(1, cfg.out_channels, H, W, device="cuda")
    plan.forward(z, out=out)   # eager pass first: nothing but the plan's own launches goes into the captures below
    plan.backward(dout)
    torch.cuda.synchronize()
    nodes = (graph_nodes(lambda: plan.forward(z, out=out)), graph_nodes(lambda: plan.backward(dout)))
    assert nodes == plan.num_launches(), "graph nodes (forward, backward) %s != dip_plan_num_launches %s" % (
        nodes, plan.num_launches())
