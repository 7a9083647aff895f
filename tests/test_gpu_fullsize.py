"""GPU parity at the BENCHMARKED configurations (BASELINE.json configs 2 and 3), full graphs, full T = 6 conv
stack, every precision the bench reports -- against the reference-equivalent fp32 torch ops on CUDA tensors
(oracle port, TF32 off).  Plus the robustness properties of the persistent application kernel."""
import numpy as np
import pytest
import torch

from oracle import nnconv_oracle as O
from tests.helpers import TOL, make_conv, oracle_stack_on_cuda, rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dev():
    assert torch.cuda.is_available()
    return torch.device('cuda:0')


def _conv_cls():
    from graph_pde_b200.nn_conv import NNConv_old
    return NNConv_old


def _darcy_case(s, r, dev, w=64, kw=1024, seed=0):
    from graph_pde_b200 import graphs
    ei = graphs.ball_connectivity(s, r, dev, True)
    x6, _, ea = graphs.darcy_sample(s, r, dev, seed=seed, edge_index=ei)
    ws, bs, root, bias = O.reference_init(w, w, [6, kw, kw, w * w], seed=0)
    torch.manual_seed(seed)
    x0 = torch.randn(s * s, w, device=dev)
    return ei, ea, x0, ws, bs, root, bias


def _run_stack(conv, x, ei, ea, depth):
    outs = []
    with torch.no_grad():
        for _ in range(depth):
            x = torch.relu(conv(x, ei, ea))
            outs.append(x)
    return outs


@pytest.mark.parametrize('precision', ['f16', 'f16x2'])
def test_config2_full_graph_full_stack(dev, precision):
    """BASELINE config 2: 85x85, r=0.10, w=64, ker_width=1024, T=6 -- the FULL graph (E = 1,466,497) and every
    one of the 6 applications against the fp32 reference ops."""
    s, r, T = 85, 0.10, 6
    ei, ea, x0, ws, bs, root, bias = _darcy_case(s, r, dev)
    assert ei.size(1) == 1466497
    conv = make_conv(_conv_cls(), ws, bs, root, bias, 'mean', 64, 64, precision, dev)
    got = _run_stack(conv, x0, ei, ea, T)
    dws, dbs = [w.to(dev) for w in ws], [b.to(dev) for b in bs]
    ref = oracle_stack_on_cuda(x0, ei, ea, dws, dbs, root.to(dev), bias.to(dev), T)
    for k in range(T):
        assert rel_err(got[k], ref[k]) < TOL[precision], (precision, k, rel_err(got[k], ref[k]))


@pytest.mark.parametrize('precision,s,n_edges', [pytest.param('f16', 241, 24557297, id='f16'),
                                                 pytest.param('f16x2', 201, 12268009, id='f16x2')])
def test_config3_full_graph_full_stack(dev, precision, s, n_edges):
    """BASELINE config 3 / the bench workload: 241x241, r=0.05 (E = 24,557,297, ties in), w=64, ker_width=1024,
    T=6.  ~30 s of fp32 reference ops on the GPU.  f16x2 keeps its edge features as fp16 pairs (4 KB per edge:
    94 GiB at 241^2, more than an 80 GB H100 holds), so it runs the largest mesh of the same family with the same
    47 GiB footprint, 201x201 (E = 12,268,009)."""
    r, T = 0.05, 6
    ei, ea, x0, ws, bs, root, bias = _darcy_case(s, r, dev, seed=3)
    assert ei.size(1) == n_edges
    conv = make_conv(_conv_cls(), ws, bs, root, bias, 'mean', 64, 64, precision, dev)
    got = _run_stack(conv, x0, ei, ea, T)
    conv._h_cache.clear()
    torch.cuda.empty_cache()
    dws, dbs = [w.to(dev) for w in ws], [b.to(dev) for b in bs]
    ref = oracle_stack_on_cuda(x0, ei, ea, dws, dbs, root.to(dev), bias.to(dev), T, edge_chunk=1 << 16)
    errs = [rel_err(got[k], ref[k]) for k in range(T)]
    assert max(errs) < TOL[precision], (precision, errs)


def test_apply_while_other_kernels_hold_sms(dev):
    """The persistent application kernel needs all its CTAs co-resident (inter-CTA flags).  It is launched
    cooperatively, so a kernel that occupies SMs on another stream (here: 100 CTAs x 200 KB of shared memory for
    30 ms, the footprint of an overlapped collective) only delays it -- the result must be the same."""
    from graph_pde_b200 import _lib
    s, r = 40, 0.12
    ei, ea, x0, ws, bs, root, bias = _darcy_case(s, r, dev, kw=256)
    conv = make_conv(_conv_cls(), ws, bs, root, bias, 'mean', 64, 64, 'f16', dev)
    with torch.no_grad():
        ref = conv(x0, ei, ea)
        torch.cuda.synchronize()
        side = torch.cuda.Stream(device=dev)
        L = _lib.lib()
        for n_ctas in (100, 148, 30):
            _lib.check(L.nnconv_debug_occupy(n_ctas, 200 * 1024, 30_000_000, side.cuda_stream))
            out = conv(x0, ei, ea)
            torch.cuda.synchronize()
            assert rel_err(out, ref) < 1e-5, n_ctas


def test_fp16_overflow_of_edge_features_is_reported(dev):
    """Hidden activations beyond the fp16 range (exotic parameter scale) must raise instead of silently turning
    into inf / NaN; bf16 handles the same parameters."""
    s, r = 12, 0.3
    ei, ea, x0, ws, bs, root, bias = _darcy_case(s, r, dev, w=32, kw=64)
    ws = [w.clone() for w in ws]
    ws[1] = ws[1] * 3.0e5                              # second hidden layer: activations ~1e6
    conv = make_conv(_conv_cls(), ws, bs, root, bias, 'mean', 32, 32, 'f16', dev)
    with pytest.raises(FloatingPointError):
        with torch.no_grad():
            conv(x0, ei, ea)
    conv_b = make_conv(_conv_cls(), ws, bs, root, bias, 'mean', 32, 32, 'bf16', dev)
    with torch.no_grad():
        out = conv_b(x0, ei, ea)
    ref = O.nnconv_forward(x0.cpu(), ei.cpu(), ea.cpu(), ws, bs, root, bias, 'mean')
    assert bool(torch.isfinite(out).all()) and rel_err(out, ref) < TOL['bf16']


def test_invalidate_after_data_write(dev):
    """Parameter writes through .data bypass the version counters the caches key on; invalidate() is the
    documented way to refresh them; normal in-place ops (what optimizers do) refresh automatically."""
    s, r = 12, 0.3
    ei, ea, x0, ws, bs, root, bias = _darcy_case(s, r, dev, w=32, kw=64)
    conv = make_conv(_conv_cls(), ws, bs, root, bias, 'mean', 32, 32, 'f16', dev)
    lin = [m for m in conv.nn.layers if isinstance(m, torch.nn.Linear)]
    with torch.no_grad():
        a = conv(x0, ei, ea)
        lin[1].weight.mul_(0.5)                        # bumps _version -> picked up
        b = conv(x0, ei, ea)
        lin[1].weight.data.mul_(2.0)                   # does not bump _version
        conv.invalidate()
        c = conv(x0, ei, ea)
    assert rel_err(b, a) > 1e-3
    assert rel_err(c, a) < 1e-6
