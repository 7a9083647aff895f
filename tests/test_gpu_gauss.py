"""The Gaussian-kernel NNConv on the H100: forward parity with the fp64 oracle for every aggregation, flow, option and
channel count (the scalar and the 16-byte paths), gradients of x, edge_attr, nn's parameters, root and bias against fp64
autograd for one and for six applications of a shared conv, exact probes bit for bit (tests/gauss_probe.py), the same
bits at every `precision`, which kernels run, the memory of a 241^2 training step, and CUDA-graph replays."""
import os

import pytest
import torch
import torch.nn.functional as F

from graph_pde_b200 import GaussianNNConv
from tests import gauss_oracle as G
from tests import gauss_probe as GP
from tests.helpers import TOL, rel_err

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _edge_attr(e, k_in, seed):
    """p0 ~ N(0, 1); p1, p2 of magnitude in [0.25, 1.25] with random signs (finite amplitudes); other columns N(0, 1)."""
    g = torch.Generator().manual_seed(seed)
    ea = torch.randn(e, k_in, generator=g)
    sign = torch.where(torch.rand(e, 2, generator=g) < 0.5, -1.0, 1.0)
    ea[:, 1:3] = (torch.rand(e, 2, generator=g) + 0.25) * sign
    return ea


def _conv(c, aggr='add', rw=True, bs=True, flow='source_to_target', precision=None, seed=0, net='linear'):
    torch.manual_seed(seed)
    nn = torch.nn.Linear(1, c) if net == 'linear' else torch.nn.Sequential(
        torch.nn.Linear(1, 16), torch.nn.ReLU(), torch.nn.Linear(16, c))
    return GaussianNNConv(c, c, nn, aggr=aggr, root_weight=rw, bias=bs, flow=flow, precision=precision).to(DEV)


def _ref_forward(conv, x, ei, ea):
    nn64 = _double_copy(conv.nn)
    sigma = nn64(torch.ones(1, dtype=torch.float64))
    root = conv.root.detach().double().cpu() if conv.root is not None else None
    bias = conv.bias.detach().double().cpu() if conv.bias is not None else None
    return G.gauss_forward(x.double().cpu(), ei.cpu(), ea.double().cpu(), sigma, root, bias, conv.aggr, conv.flow)


def _double_copy(nn):
    import copy
    return copy.deepcopy(nn).cpu().double()


@pytest.mark.parametrize('aggr', ['add', 'mean', 'max'])
@pytest.mark.parametrize('c', [1, 16, 64, 128])
@pytest.mark.parametrize('k_in', [3, 6])
def test_forward_matches_oracle(aggr, c, k_in):
    ei = GP.graph(seed=c + k_in)
    ea = _edge_attr(ei.size(1), k_in, seed=c)
    x = torch.randn(300, c, generator=torch.Generator().manual_seed(c))
    for rw, bs, flow in ((True, True, 'source_to_target'), (False, False, 'source_to_target'),
                         (True, False, 'target_to_source'), (False, True, 'target_to_source')):
        conv = _conv(c, aggr, rw, bs, flow, seed=c)
        with torch.no_grad():
            out = conv(x.to(DEV), ei.to(DEV), ea.to(DEV))
        ref, _ = _ref_forward(conv, x, ei, ea)
        assert rel_err(out, ref) < TOL['fp32'], (aggr, c, k_in, rw, bs, flow, rel_err(out, ref))


def test_unaligned_x_and_1d_input():
    """An x that starts off a 16-byte boundary runs the scalar path with the same result; 1-D x is unsqueezed."""
    ei = GP.graph(seed=3).to(DEV)
    ea = _edge_attr(ei.size(1), 3, seed=3).to(DEV)
    conv = _conv(64, 'mean')
    buf = torch.randn(300 * 64 + 1, device=DEV)
    x_un = buf[1:].view(300, 64)
    with torch.no_grad():
        out_un = conv(x_un, ei, ea)
        out_al = conv(x_un.clone(), ei, ea)
    assert rel_err(out_un, out_al) < 1e-6
    conv1 = _conv(1, 'add')
    x1 = torch.randn(300, device=DEV)
    with torch.no_grad():
        out1 = conv1(x1, ei, ea)
    ref1, _ = _ref_forward(conv1, x1.unsqueeze(-1), ei, ea)
    assert out1.shape == (300, 1) and rel_err(out1, ref1) < TOL['fp32']


def _grads_vs_oracle(aggr, T, c=64, net='mlp', k_in=6, flow='source_to_target', seed=0):
    """KernelNN-style chain h <- relu(conv(h)) T times through one shared conv; every gradient against fp64 autograd
    through the oracle.  The edge_attr gradient of an edge sums C channel terms that largely cancel, and through six
    fp32 applications whose values grow to ~1e5 its error relative to the largest entry reaches a few 1e-4 (measured
    2.3e-4 for add and max on an H100): T = 6 is held to 1e-3, T <= 2 to 1e-4."""
    ei = GP.graph(seed=seed)
    ea = _edge_attr(ei.size(1), k_in, seed=seed) * 0.5
    ea[:, 1:3] = ea[:, 1:3].sign() * (ea[:, 1:3].abs() + 0.5)
    x = torch.randn(300, c, generator=torch.Generator().manual_seed(seed)) * 0.5
    gout = torch.randn(300, c, generator=torch.Generator().manual_seed(seed + 1))
    conv = _conv(c, aggr, flow=flow, seed=seed, net=net)
    xd, ead = x.to(DEV).requires_grad_(), ea.to(DEV).requires_grad_()
    h = xd
    for _ in range(T):
        h = F.relu(conv(h, ei.to(DEV), ead))
    (h * gout.to(DEV)).sum().backward()

    nn64 = _double_copy(conv.nn)
    for p in nn64.parameters():
        p.requires_grad_()
    root = conv.root.detach().double().cpu().requires_grad_()
    bias = conv.bias.detach().double().cpu().requires_grad_()
    x64, ea64 = x.double().requires_grad_(), ea.double().requires_grad_()
    h64 = x64
    for _ in range(T):
        sigma = nn64(torch.ones(1, dtype=torch.float64))
        h64 = F.relu(G.gauss_forward(h64, ei, ea64, sigma, root, bias, aggr, flow)[0])
    (h64 * gout.double()).sum().backward()
    pairs = [('x', xd.grad, x64.grad), ('edge_attr', ead.grad, ea64.grad), ('root', conv.root.grad, root.grad),
             ('bias', conv.bias.grad, bias.grad)]
    pairs += [('nn.' + k, p.grad, q.grad) for (k, p), q in zip(conv.nn.named_parameters(), nn64.parameters())]
    tol = 1e-4 if T <= 2 else 1e-3
    for name, got, want in pairs:
        assert got is not None, name
        assert rel_err(got, want) < tol, (aggr, T, name, rel_err(got, want))


@pytest.mark.parametrize('aggr', ['add', 'mean', 'max'])
@pytest.mark.parametrize('T', [1, 6])
def test_gradients_match_fp64_autograd(aggr, T):
    _grads_vs_oracle(aggr, T, net='mlp' if T == 6 else 'linear', k_in=6 if T == 6 else 3, seed=T)


@pytest.mark.parametrize('c', [1, 16, 128])
def test_gradients_other_channel_counts(c):
    _grads_vs_oracle('mean', 2, c=c, net='linear', k_in=3, flow='target_to_source', seed=c)


@pytest.mark.parametrize('aggr', ['add', 'max'])
@pytest.mark.parametrize('flow', ['source_to_target', 'target_to_source'])
@pytest.mark.parametrize('k_in', [3, 6])
@pytest.mark.parametrize('c', [16, 64])
def test_exact_probe_bit_for_bit(aggr, flow, k_in, c):
    """Forward, argmax and every gradient equal fp64 autograd through the oracle exactly (tests/gauss_probe.py);
    under max, ties go to the smallest caller edge and the gradient to the winner only."""
    ei = GP.graph(seed=7)
    ea = GP.edge_attr(ei.size(1), k_in, seed=7)
    x, gout, root, bias = GP.tensors(300, c, seed=7)
    lin = GP.nn_module(c, seed=7)
    out64, am64, g64 = GP.reference(x, ei, ea, lin, root, bias, gout, aggr, torch.float64, flow)
    conv = GaussianNNConv(c, c, torch.nn.Linear(1, c), aggr=aggr, flow=flow).to(DEV)
    conv.nn.load_state_dict(lin.state_dict())
    with torch.no_grad():
        conv.root.copy_(root)
        conv.bias.copy_(bias)
    xd, ead = x.float().to(DEV).requires_grad_(), ea.float().to(DEV).requires_grad_()
    out = conv(xd, ei.to(DEV), ead)
    (out * gout.float().to(DEV)).sum().backward()
    assert torch.equal(out.detach().double().cpu(), out64)
    got = {'x': xd.grad, 'edge_attr': ead.grad, 'nn.weight': conv.nn.weight.grad, 'nn.bias': conv.nn.bias.grad,
           'root': conv.root.grad, 'bias': conv.bias.grad}
    for k, v in g64.items():
        assert torch.equal(got[k].double().cpu(), v), (k, (got[k].double().cpu() - v).abs().max())
    if aggr == 'max':
        from graph_pde_b200.nn_conv import get_plan
        with torch.no_grad():
            plan = get_plan(ei.to(DEV), 300, flow)
            _, argmax = conv._apply_impl(plan, xd.detach(), ead.detach(), conv._sigma(DEV).detach())
        assert torch.equal(argmax.long().cpu(), am64)
        assert (am64 >= 0).sum() > 0 and ((am64 == -1).all(dim=1) | (am64 >= 0).all(dim=1)).all()


def test_precision_values_give_identical_bits(monkeypatch):
    """Every `precision` (and NNCONV_B200_PRECISION) computes the same fp32 result.  Compared where the result does not
    depend on the order of the fp32 atomics: add on the exact probe without root and bias, max on random data."""
    ei = GP.graph(seed=9).to(DEV)
    cases = [('add', GP.edge_attr(ei.size(1), 6, seed=9).float(), GP.tensors(300, 64, seed=9)[0].float()),
             ('max', _edge_attr(ei.size(1), 6, seed=9), torch.randn(300, 64))]
    for aggr, ea, x in cases:
        ea, x = ea.to(DEV), x.to(DEV)
        outs = []
        for prec in ('f16', 'bf16', 'f16x2', 'fp32', None):
            conv = _conv(64, aggr, rw=aggr == 'max', bs=aggr == 'max', precision=prec, seed=9)
            if aggr == 'add':
                conv.nn.load_state_dict(GP.nn_module(64, seed=9).state_dict())
            with torch.no_grad():
                outs.append(conv(x, ei, ea))
        with monkeypatch.context() as m:
            m.setenv('NNCONV_B200_PRECISION', 'bf16')
            with torch.no_grad():
                outs.append(conv(x, ei, ea))
        for o in outs[1:]:
            assert torch.equal(o, outs[0]), aggr


_NAMES_SCRIPT = r"""
import sys, time, torch
sys.path.insert(0, %r)
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile
from graph_pde_b200 import GaussianNNConv
from tests.gauss_probe import graph
aggr = sys.argv[1]
ei = graph(seed=1).cuda()
conv = GaussianNNConv(64, 64, torch.nn.Linear(1, 64), aggr=aggr, root_weight=False).cuda()
x = torch.randn(300, 64, device='cuda', requires_grad=True)
ea = torch.rand(ei.size(1), 6, device='cuda').add_(0.5).requires_grad_()
conv(x, ei, ea).square().sum().backward()
torch.cuda.synchronize()
for _ in range(4):
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        conv(x, ei, ea).square().sum().backward()
        torch.cuda.synchronize()
        time.sleep(0.02)
    names = {e.name for e in prof.events() if e.device_type == DeviceType.CUDA}
    if names:
        break
print('NAMES', ' | '.join(sorted(names)))
""" % ROOT


@pytest.mark.parametrize('aggr', ['mean', 'max'])
def test_profiler_shows_the_fused_kernels(aggr):
    """One forward and backward launch k_apply_gauss and k_bwd_gauss and none of the library's GEMMs or d builds."""
    import subprocess
    import sys
    res = subprocess.run([sys.executable, '-c', _NAMES_SCRIPT, aggr], cwd=ROOT, stdout=subprocess.PIPE,
                         stderr=subprocess.STDOUT, text=True, timeout=600)
    assert res.returncode == 0 and 'NAMES' in res.stdout, res.stdout
    names = res.stdout.split('NAMES', 1)[1]
    assert 'k_apply_gauss' in names and 'k_bwd_gauss' in names, names
    lib_names = [n for n in names.split(' | ') if 'nnc::' in n]
    for bad in ('gemm', 'k_diag_build', 'k_apply_diag', 'k_bwd_diag', 'k_conv', 'k_apply_tc'):
        assert not any(bad in n for n in lib_names), (bad, lib_names)


def test_memory_at_241_is_below_one_edge_channel_tensor():
    """At 241^2, r = 0.05 one forward and backward raise the peak allocation by less than one [E, 64] fp32 tensor."""
    from graph_pde_b200 import graphs
    x6, ei, ea = graphs.darcy_sample(241, 0.05, device=DEV)
    E = ei.size(1)
    ea = ea.clone()
    ea[:, 1:3] = ea[:, 1:3].abs() + 0.5
    conv = _conv(64, 'mean')
    x = torch.randn(x6.size(0), 64, device=DEV, requires_grad=True)
    ea.requires_grad_()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(DEV)
    torch.cuda.reset_peak_memory_stats(DEV)
    out = conv(x, ei, ea)
    out.square().mean().backward()
    torch.cuda.synchronize()
    rise = torch.cuda.max_memory_allocated(DEV) - base
    assert torch.isfinite(x.grad).all() and torch.isfinite(conv.nn.weight.grad).all()
    assert rise < E * 64 * 4, (rise, E * 64 * 4)


class _KernelNNGauss(torch.nn.Module):
    def __init__(self, c, k_in, T):
        super().__init__()
        self.fc1 = torch.nn.Linear(6, c)
        self.conv = GaussianNNConv(c, c, torch.nn.Sequential(torch.nn.Linear(1, 16), torch.nn.ReLU(),
                                                             torch.nn.Linear(16, c)), aggr='mean')
        self.fc2 = torch.nn.Linear(c, 1)
        self.T = T

    def forward(self, x, ei, ea):
        h = self.fc1(x)
        for _ in range(self.T):
            h = F.relu(self.conv(h, ei, ea))
        return self.fc2(h)


def test_graphed_forward_replay():
    from graph_pde_b200 import GraphedForward
    torch.manual_seed(0)
    model = _KernelNNGauss(32, 6, 3).to(DEV)
    ei = GP.graph(seed=11).to(DEV)
    ea = _edge_attr(ei.size(1), 6, seed=11).to(DEV)
    x = torch.randn(300, 6, device=DEV)
    gf = GraphedForward(model, x, ei, ea)
    x.copy_(torch.randn(300, 6, device=DEV))
    out = gf.replay().clone()
    with torch.no_grad():
        ref = model(x, ei, ea)
    assert rel_err(out, ref) < 1e-6


def test_graphed_train_step_replay_equals_eager():
    from graph_pde_b200 import GraphedTrainStep
    ei = GP.graph(seed=12).to(DEV)
    ea = _edge_attr(ei.size(1), 6, seed=12).to(DEV)
    x = torch.randn(300, 6, device=DEV)
    y = torch.randn(300, 1, device=DEV)
    torch.manual_seed(0)
    model_e, model_g = _KernelNNGauss(32, 6, 3).to(DEV), _KernelNNGauss(32, 6, 3).to(DEV)
    model_g.load_state_dict(model_e.state_dict())
    opt_e = torch.optim.Adam(model_e.parameters(), lr=1e-3, capturable=True)
    opt_g = torch.optim.Adam(model_g.parameters(), lr=1e-3, capturable=True)
    xg, eag, yg = x.clone(), ea.clone(), y.clone()
    step = GraphedTrainStep(lambda a, b, c: F.mse_loss(model_g(a, ei, b), c), model_g, opt_g, xg, eag, yg)
    for i in range(5):
        opt_e.zero_grad(set_to_none=True)
        loss_e = F.mse_loss(model_e(x, ei, ea), y)
        loss_e.backward()
        opt_e.step()
        loss_g = step.replay()
        assert abs(float(loss_g) - float(loss_e)) <= 1e-4 * max(1.0, abs(float(loss_e))), (i, float(loss_g), float(loss_e))
    for (k, a), b in zip(model_e.state_dict().items(), model_g.state_dict().values()):
        assert rel_err(b, a) < 1e-4, k
    with torch.no_grad():
        assert rel_err(model_g(x, ei, ea), model_e(x, ei, ea)) < 1e-4
