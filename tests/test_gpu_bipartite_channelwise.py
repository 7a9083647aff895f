"""Bipartite DiagNNConv and GaussianNNConv on the H100 (DESIGN 4.10): messages from x_src into the rows of x_dst.

* forward parity against the fp64 restatement (tests/bipartite_channelwise_oracle.py) at every precision and
  aggregation, for N_src > N_dst and N_src < N_dst, with sources without out-edges and targets without in-edges;
  x_dst = None with size, and no root or bias;
* union equivalence bit for bit on exact integer probes: the bipartite output and every gradient equal the square
  conv's on the union graph [x_src; x_dst] with edges (src, N_src + dst), whose output gradient is zero on the source
  rows (in-degrees are powers of two, so aggr='mean' stays exact too);
* gradients against fp64 autograd for T = 1 and 3 pairs over one graph (DiagNNConv: one edge-network pass for all);
* the kernels that run, CUDA-graph replay of a forward and of a training step, the drop-in classes and the refusals."""
import os
import subprocess
import sys

import pytest
import torch

from tests import bipartite_channelwise_oracle as O
from tests import gauss_probe as GP
from tests.helpers import TOL, rel_err
from tests.test_gpu_bipartite import bip_graph, pow2_bip_graph

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
PRECS = ['f16', 'bf16', 'f16x2', 'fp32']
AGGRS = ['add', 'mean', 'max']
KINDS = ['diag', 'gauss']
C, KIN = 64, 3


def make_conv(kind, aggr, precision, seed=0, root_weight=True, bias=True, **kw):
    from graph_pde_b200.gauss import GaussianNNConv
    from graph_pde_b200.nn_conv import DiagNNConv
    torch.manual_seed(seed)
    if kind == 'diag':
        nn = torch.nn.Sequential(torch.nn.Linear(KIN, 64), torch.nn.ReLU(), torch.nn.Linear(64, C))
        conv = DiagNNConv(C, C, nn, aggr=aggr, precision=precision, root_weight=root_weight, bias=bias, **kw)
    else:
        nn = torch.nn.Sequential(torch.nn.Linear(1, 16), torch.nn.ReLU(), torch.nn.Linear(16, C))
        conv = GaussianNNConv(C, C, nn, aggr=aggr, precision=precision, root_weight=root_weight, bias=bias, **kw)
    return conv.to(DEV)


def edge_attr(e, seed=1):
    """|p1 p2| >= 1/16: finite Gaussian amplitudes."""
    g = torch.Generator().manual_seed(seed)
    sign = torch.where(torch.rand(e, KIN, generator=g) < 0.5, -1.0, 1.0)
    return (torch.rand(e, KIN, generator=g) + 0.25) * sign


def node_inputs(n_src, n_dst, seed=2, T=1):
    g = torch.Generator().manual_seed(seed)
    return ([torch.randn(n_src, C, generator=g) for _ in range(T)], [torch.randn(n_dst, C, generator=g) for _ in range(T)])


def ref_d(conv, ea):
    """The fp64 diagonal [E, C] of ``conv`` on ``ea`` (differentiable w.r.t. ea and, as given, the parameters)."""
    from graph_pde_b200.nn_conv import DiagNNConv
    if isinstance(conv, DiagNNConv):
        lin = [conv.nn[0], conv.nn[2]]
        return O.diag_d(ea, [l.weight.detach().double().to(ea.device) for l in lin],
                        [l.bias.detach().double().to(ea.device) for l in lin])
    nn64 = _double_copy(conv.nn).to(ea.device)
    return O.gauss_d(ea, nn64(torch.ones(1, dtype=torch.float64, device=ea.device)))


def _double_copy(m):
    import copy
    return copy.deepcopy(m).double()


def oracle(conv, x_src, x_dst, ei, ea, n_dst):
    dev = x_src.device
    d = ref_d(conv, ea.double().to(dev))
    root = None if conv.root is None else conv.root.detach().double()
    bias = None if conv.bias is None else conv.bias.detach().double()
    return O.forward(x_src.double(), None if x_dst is None else x_dst.double().to(dev), ei.to(dev), d, root, bias,
                     conv.aggr, n_dst)[0]


def run(conv, x_src, x_dst, ei, ea, size=None):
    with torch.no_grad():
        return conv((x_src.to(DEV), None if x_dst is None else x_dst.to(DEV)), ei.to(DEV), ea.to(DEV), size=size)


def tol_of(kind, precision):
    return TOL[precision] if kind == 'diag' else TOL['fp32']    # the Gaussian conv is fp32 at every precision


# ---- forward parity -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('precision', PRECS)
@pytest.mark.parametrize('aggr', AGGRS)
@pytest.mark.parametrize('shape', [(700, 300, 6000), (250, 900, 5000)])
@pytest.mark.parametrize('kind', KINDS)
def test_forward_parity(kind, shape, aggr, precision):
    n_src, n_dst, e = shape
    ei = bip_graph(n_src, n_dst, e)
    ea = edge_attr(e)
    (xs,), (xd,) = node_inputs(n_src, n_dst)
    conv = make_conv(kind, aggr, precision)
    out = run(conv, xs, xd, ei, ea)
    assert out.shape == (n_dst, C)
    ref = oracle(conv, xs.to(DEV), xd, ei, ea, n_dst)
    assert rel_err(out, ref) < tol_of(kind, precision), (kind, shape, aggr, precision, rel_err(out, ref))
    root_term = xd[:2].to(DEV) @ conv.root.detach() + conv.bias.detach()           # targets 0, 1: no in-edges
    assert float((out[:2] - root_term).abs().max()) < 1e-5


@pytest.mark.parametrize('aggr', AGGRS)
@pytest.mark.parametrize('kind', KINDS)
def test_forward_options(kind, aggr):
    """x_dst = None with size (both forms), root_weight=False and bias=False."""
    n_src, n_dst = 300, 500
    ei = bip_graph(n_src, n_dst, 3000)
    ea = edge_attr(3000)
    (xs,), (xd,) = node_inputs(n_src, n_dst)
    conv = make_conv(kind, aggr, 'f16x2')
    for size in ((n_src, n_dst), (None, n_dst)):
        out = run(conv, xs, None, ei, ea, size=size)
        assert rel_err(out, oracle(conv, xs.to(DEV), None, ei, ea, n_dst)) < TOL['f16x2'], size
    for rw, b in ((False, True), (True, False), (False, False)):
        conv = make_conv(kind, aggr, 'f16x2', root_weight=rw, bias=b)
        out = run(conv, xs, xd, ei, ea, size=(n_src, n_dst))
        assert rel_err(out, oracle(conv, xs.to(DEV), xd, ei, ea, n_dst)) < TOL['f16x2'], (rw, b)


# ---- union equivalence, bit for bit --------------------------------------------------------------------------------------
def probe_conv(kind, aggr, precision, seed):
    """A conv whose every weight is a small integer (DiagNNConv: tests/test_gpu_diag.py's probe layers; GaussianNNConv:
    tests/gauss_probe.py's sigma of small nonzero integers), with an integer root and bias."""
    from graph_pde_b200.gauss import GaussianNNConv
    from graph_pde_b200.nn_conv import DiagNNConv
    from tests.test_gpu_diag import _probe_layers
    g = torch.Generator().manual_seed(seed)
    if kind == 'diag':
        conv = DiagNNConv(C, C, torch.nn.Sequential(torch.nn.Linear(KIN, 64), torch.nn.ReLU(), torch.nn.Linear(64, C)),
                          aggr=aggr, precision=precision)
        with torch.no_grad():
            for lin, (w, b) in zip([conv.nn[0], conv.nn[2]], _probe_layers(seed)):
                lin.weight.copy_(w)
                lin.bias.copy_(b)
    else:
        conv = GaussianNNConv(C, C, torch.nn.Linear(1, C), aggr=aggr, precision=precision)
        conv.nn.load_state_dict(GP.nn_module(C, seed).state_dict())    # after the constructor's reset of nn
    with torch.no_grad():
        conv.root.copy_(torch.randint(-1, 2, (C, C), generator=g).float())
        conv.bias.copy_(torch.randint(-2, 3, (C,), generator=g).float())
    return conv.to(DEV)


def probe_edge_attr(kind, e, seed):
    if kind == 'diag':
        return torch.randint(-2, 3, (e, KIN), generator=torch.Generator().manual_seed(seed)).float()
    return GP.edge_attr(e, KIN, seed).float()          # p0 = 0, |p1 p2| a power of four: every message exact


def _grads(conv, out, g, tensors):
    for q in conv.parameters():
        q.grad = None
    out.backward(g)
    return [t.grad.clone() for t in tensors] + [q.grad.clone() for q in conv.parameters()]


@pytest.mark.parametrize('precision', PRECS)
@pytest.mark.parametrize('aggr', AGGRS)
@pytest.mark.parametrize('n_src,n_dst', [(700, 260), (180, 650)])
@pytest.mark.parametrize('kind', KINDS)
def test_union_equivalence_bit_for_bit(kind, n_src, n_dst, aggr, precision):
    ei = pow2_bip_graph(n_src, n_dst, 13)
    union = torch.stack([ei[0], ei[1] + n_src]).to(DEV)
    e = ei.size(1)
    gen = torch.Generator().manual_seed(17)
    x = torch.randint(-4, 5, (n_src + n_dst, C), generator=gen).float().to(DEV)
    g = torch.randint(-3, 4, (n_src + n_dst, C), generator=gen).float().to(DEV)
    g[:n_src] = 0                                  # the union's source rows are not part of the bipartite map
    ea = probe_edge_attr(kind, e, 19).to(DEV)
    conv = probe_conv(kind, aggr, precision, 23)
    xu, eau = x.clone().requires_grad_(), ea.clone().requires_grad_()
    out_u = conv(xu, union, eau)
    gu = _grads(conv, out_u, g, [xu, eau])
    xs, xd = x[:n_src].clone().requires_grad_(), x[n_src:].clone().requires_grad_()
    eab = ea.clone().requires_grad_()
    out_b = conv((xs, xd), ei.to(DEV), eab)
    assert out_b.shape == (n_dst, C)
    assert torch.equal(out_b, out_u[n_src:]), float((out_b - out_u[n_src:]).abs().max())
    ref = oracle(conv, x[:n_src], x[n_src:], ei, ea, n_dst)
    assert torch.equal(out_b.double(), ref), float((out_b.double() - ref).abs().max())     # and exact
    gb = _grads(conv, out_b, g[n_src:], [xs, xd, eab])
    assert torch.equal(gb[0], gu[0][:n_src]), 'dx_src'
    assert torch.equal(gb[1], gu[0][n_src:]), 'dx_dst'
    assert torch.equal(gb[2], gu[1]), 'd edge_attr'
    for (name, _), a, b in zip(conv.named_parameters(), gb[3:], gu[2:]):
        assert torch.equal(a, b), name


# ---- gradients against fp64 autograd --------------------------------------------------------------------------------
@pytest.mark.parametrize('aggr', AGGRS)
@pytest.mark.parametrize('T', [1, 3])
@pytest.mark.parametrize('kind', KINDS)
def test_grads_against_fp64(kind, T, aggr):
    from graph_pde_b200 import nn_conv
    n_src, n_dst = 400, 700
    ei = bip_graph(n_src, n_dst, 5000)
    ea = edge_attr(5000)
    xs, xd = node_inputs(n_src, n_dst, T=T)
    gs = [torch.randn(n_dst, C, generator=torch.Generator().manual_seed(30 + t)) for t in range(T)]
    conv = make_conv(kind, aggr, 'f16x2' if kind == 'diag' else 'fp32')
    pairs = [(a.to(DEV).requires_grad_(), b.to(DEV).requires_grad_()) for a, b in zip(xs, xd)]
    eag = ea.to(DEV).requires_grad_()
    eid = ei.to(DEV)                     # one edge_index tensor: the applications share one plan and one d
    b0, m0 = nn_conv.stats['backwards'], nn_conv.stats['mlp_backwards']
    loss = 0
    for (a, b), g in zip(pairs, gs):
        loss = loss + (conv((a, b), eid, eag) * g.to(DEV)).sum()
    loss.backward()
    assert nn_conv.stats['backwards'] == b0 + T
    if kind == 'diag':
        assert nn_conv.stats['mlp_backwards'] == m0 + 1          # the T pairs share one pass through the edge network
    # fp64 autograd
    from graph_pde_b200.nn_conv import DiagNNConv
    nn64 = _double_copy(conv.nn).to(DEV)
    for p in nn64.parameters():
        p.grad = None
        p.requires_grad_()
    root = conv.root.detach().double().requires_grad_()
    bias = conv.bias.detach().double().requires_grad_()
    ea64 = ea.double().to(DEV).requires_grad_()
    refs = [(a.double().to(DEV).requires_grad_(), b.double().to(DEV).requires_grad_()) for a, b in zip(xs, xd)]
    if isinstance(conv, DiagNNConv):
        d = nn64(ea64)
    else:
        d = O.gauss_d(ea64, nn64(torch.ones(1, dtype=torch.float64, device=DEV)))
    loss = 0
    for (a, b), g in zip(refs, gs):
        loss = loss + (O.forward(a, b, ei.to(DEV), d, root, bias, aggr, n_dst)[0] * g.double().to(DEV)).sum()
    loss.backward()
    tol = 2e-4
    for (a, b), (ra, rb) in zip(pairs, refs):
        assert rel_err(a.grad, ra.grad) < tol, 'x_src'
        assert rel_err(b.grad, rb.grad) < tol, 'x_dst'
    assert rel_err(conv.root.grad, root.grad) < tol, 'root'
    assert rel_err(conv.bias.grad, bias.grad) < tol, 'bias'
    for (name, p), q in zip(conv.nn.named_parameters(), nn64.parameters()):
        assert rel_err(p.grad, q.grad) < 1e-3, name
    assert rel_err(eag.grad, ea64.grad) < 1e-3, 'edge_attr'


@pytest.mark.parametrize('kind', KINDS)
def test_x_dst_none_and_x_dst_dtype(kind):
    n_src, n_dst = 300, 200
    ei = bip_graph(n_src, n_dst, 2000).to(DEV)
    ea = edge_attr(2000).to(DEV)
    (xs,), (xd,) = node_inputs(n_src, n_dst)
    conv = make_conv(kind, 'add', 'f16x2')
    x = xs.to(DEV).requires_grad_()
    conv((x, None), ei, ea, size=(n_src, n_dst)).sum().backward()
    assert torch.equal(conv.root.grad, torch.zeros_like(conv.root))
    assert torch.allclose(conv.bias.grad, torch.full_like(conv.bias, float(n_dst)))
    assert x.grad is not None and torch.isfinite(x.grad).all()
    xd64 = xd.double().to(DEV).requires_grad_()                 # x_dst's gradient comes back in x_dst's dtype
    conv((xs.to(DEV), xd64), ei, ea).sum().backward()
    assert xd64.grad.dtype == torch.float64
    ref = torch.ones(n_dst, C, dtype=torch.float64, device=DEV) @ conv.root.detach().double().t()
    assert rel_err(xd64.grad, ref) < 1e-6


# ---- which kernels run --------------------------------------------------------------------------------------------------
_NAMES_SCRIPT = """
import sys, time, torch
sys.path.insert(0, %r)
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile
from tests.test_gpu_bipartite import bip_graph
from tests.test_gpu_bipartite_channelwise import edge_attr, make_conv, node_inputs
kind, precision = sys.argv[1], sys.argv[2]
n_src, n_dst = 500, 800
ei = bip_graph(n_src, n_dst, 4000).cuda()
ea = edge_attr(4000).cuda().requires_grad_()
(xs,), (xd,) = node_inputs(n_src, n_dst)
xs, xd = xs.cuda(), xd.cuda()
union = torch.stack([ei[0], ei[1] + n_src])
xu = torch.cat([xs, xd])
for which in ('square', 'bipartite'):
    conv = make_conv(kind, 'mean', precision)
    def step():
        if hasattr(conv, 'invalidate'):
            conv.invalidate()
        if which == 'square':
            x = xu.clone().requires_grad_()
            conv(x, union, ea).sum().backward()
        else:
            a, b = xs.clone().requires_grad_(), xd.clone().requires_grad_()
            conv((a, b), ei, ea).sum().backward()
    step()
    torch.cuda.synchronize()
    for _ in range(4):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step()
            torch.cuda.synchronize()
            time.sleep(0.02)
        names = {e.name for e in prof.events() if e.device_type == DeviceType.CUDA}
        if names:
            break
    print('NAMES', which, '|'.join(sorted(names)))
"""


@pytest.mark.parametrize('kind,precision', [('diag', 'f16'), ('diag', 'fp32'), ('gauss', 'fp32')])
def test_bipartite_runs_the_square_kernels(kind, precision):
    """A bipartite training step runs the square conv's message kernels plus the root term's: no other path."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, '-c', _NAMES_SCRIPT % root, kind, precision], cwd=root,
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert res.returncode == 0, res.stdout
    names = {l.split(' ', 2)[1]: set(l.split(' ', 2)[2].split('|')) for l in res.stdout.splitlines()
             if l.startswith('NAMES ')}
    strip = lambda s: {n.replace('(anonymous namespace)::', '').split('(')[0] for n in s}   # noqa: E731
    sq, bp = strip(names['square']), strip(names['bipartite'])
    want = ('k_apply_diag', 'k_bwd_diag_edges') if kind == 'diag' else ('k_apply_gauss', 'k_bwd_gauss')
    for k in want:
        assert any(k in n for n in bp), (k, bp)
    hot = {n for n in sq if any(k in n for k in want + ('k_diag_build', 'k_gemm_tc', 'k_max_finalize'))}
    assert hot <= bp, hot - bp
    assert any('k_root_add' in n for n in bp), bp
    # beyond the square step's kernels only the root term's (k_root_add; k_xtv, k_g_rootT, k_colsum for its backward)
    # and torch's own elementwise / reduction kernels may run
    root_term = ('k_root_add', 'k_xtv', 'k_g_rootT', 'k_colsum')
    extra = {n for n in bp - sq if not any(k in n for k in root_term) and
             not any(k in n.lower() for k in ('elementwise', 'memset', 'fill', 'reduce', 'copy'))}
    assert not extra, extra


# ---- CUDA graphs ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', KINDS)
def test_graphed_forward_with_a_bipartite_conv(kind):
    from graph_pde_b200 import GraphedForward
    n_src, n_dst = 400, 700
    ei = bip_graph(n_src, n_dst, 5000).to(DEV)
    ea = edge_attr(5000).to(DEV)
    (xs, xs2), (xd, xd2) = node_inputs(n_src, n_dst, T=2)
    xs, xd = xs.to(DEV), xd.to(DEV)
    conv = make_conv(kind, 'max', 'f16')

    class Wrap(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.conv = conv

        def forward(self, a, b, ei_, ea_):
            return self.conv((a, b), ei_, ea_)
    gf = GraphedForward(Wrap(), xs, xd, ei, ea)
    xs.copy_(xs2.to(DEV))
    xd.copy_(xd2.to(DEV))
    out = gf.replay().clone()
    with torch.no_grad():
        ref = conv((xs2.to(DEV), xd2.to(DEV)), ei, ea)
    assert out.shape == (n_dst, C)
    assert rel_err(out, ref) < 1e-6


class Decoder(torch.nn.Module):
    """Two square DiagNNConv layers on the input mesh, then a bipartite DiagNNConv and a bipartite GaussianNNConv from
    the mesh to query points."""

    def __init__(self):
        super().__init__()
        torch.manual_seed(0)
        self.fc = torch.nn.Linear(3, C)
        self.conv = make_conv('diag', 'mean', 'f16x2')
        self.dec = make_conv('diag', 'mean', 'f16x2', seed=1)
        self.gdec = make_conv('gauss', 'add', 'fp32', seed=2)
        self.q = torch.nn.Linear(2, C)
        self.out = torch.nn.Linear(C, 1)

    def forward(self, x, ei, ea, qpos, ei_q, ea_q):
        h = self.fc(x)
        for _ in range(2):
            h = torch.relu(self.conv(h, ei, ea))
        q = self.q(qpos)
        y = torch.relu(self.dec((h, q), ei_q, ea_q)) + 0.1 * self.gdec((h, q), ei_q, ea_q)
        return self.out(y).view(-1)


def test_graphed_train_step_with_bipartite_channelwise_convs():
    import torch.nn.functional as F
    from graph_pde_b200 import GraphedTrainStep
    n, m = 400, 600
    g = torch.Generator().manual_seed(5)
    ei = torch.stack([torch.randint(0, n, (4000,), generator=g), torch.randint(0, n, (4000,), generator=g)])
    ei_q = bip_graph(n, m, 5000, seed=6)
    data = [torch.randn(n, 3, generator=g), ei, edge_attr(4000, seed=7), torch.rand(m, 2, generator=g), ei_q,
            edge_attr(5000, seed=8)]
    y = torch.randn(m, generator=g)
    data = [t.to(DEV) for t in data]
    y = y.to(DEV)
    mg, me = Decoder().to(DEV), Decoder().to(DEV)
    me.load_state_dict(mg.state_dict())
    og = torch.optim.Adam(mg.parameters(), lr=1e-3, capturable=True)
    oe = torch.optim.Adam(me.parameters(), lr=1e-3, capturable=True)
    step = GraphedTrainStep(lambda *a: F.mse_loss(mg(*a[:-1]), a[-1]), mg, og, *data, y)
    tol = 1e-4
    for k in range(3):
        loss_g = float(step.replay())
        oe.zero_grad()
        loss_e = F.mse_loss(me(*data), y)
        loss_e.backward()
        oe.step()
        assert abs(loss_g - float(loss_e)) <= tol * max(1.0, abs(float(loss_e))), (k, loss_g, float(loss_e))
        for (name, a), b in zip(mg.named_parameters(), me.parameters()):
            assert rel_err(a.detach(), b.detach()) < tol, (k, name)


# ---- the drop-in classes and the refusals ---------------------------------------------------------------------------------
def test_dropin_classes_take_the_pair():
    import importlib.util
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location('dropin_nn_conv', os.path.join(root, 'dropin', 'nn_conv.py'))
    dropin = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(dropin)
    n_src, n_dst = 300, 200
    ei = bip_graph(n_src, n_dst, 2000)
    ea = edge_attr(2000)
    (xs,), (xd,) = node_inputs(n_src, n_dst)
    for kind, cls in (('diag', dropin.NNConv), ('gauss', dropin.NNConv_Gaussian)):
        lib = make_conv(kind, 'mean', 'fp32')
        torch.manual_seed(0)
        nn = (torch.nn.Sequential(torch.nn.Linear(KIN, 64), torch.nn.ReLU(), torch.nn.Linear(64, C)) if kind == 'diag'
              else torch.nn.Sequential(torch.nn.Linear(1, 16), torch.nn.ReLU(), torch.nn.Linear(16, C)))
        conv = cls(C, C, nn, aggr='mean', precision='fp32').to(DEV)
        conv.load_state_dict(lib.state_dict())
        out = run(conv, xs, xd, ei, ea)
        assert rel_err(out, run(lib, xs, xd, ei, ea)) < 1e-6, kind


@pytest.mark.parametrize('kind', KINDS)
def test_host_refusals_launch_nothing(kind):
    from graph_pde_b200 import nn_conv
    ei = bip_graph(50, 30, 200).to(DEV)
    ea = edge_attr(200).to(DEV)
    xs, xd = torch.randn(50, C, device=DEV), torch.randn(30, C, device=DEV)
    launches, applies = nn_conv.stats['launches'], nn_conv.stats['applies']
    conv = make_conv(kind, 'add', 'f16', flow='target_to_source')
    with pytest.raises(ValueError, match='target_to_source'):
        conv((xs, xd), ei, ea)
    conv = make_conv(kind, 'add', 'f16')
    with pytest.raises(ValueError, match='size'):
        conv((xs, None), ei, ea)
    with pytest.raises(ValueError, match='disagrees'):
        conv((xs, xd), ei, ea, size=(50, 31))
    with pytest.raises(ValueError, match='x_dst has shape'):
        conv((xs, torch.randn(30, 8, device=DEV)), ei, ea)
    with pytest.raises(ValueError, match='x_dst has shape'):
        conv((xs, torch.randn(30, C, 1, device=DEV)), ei, ea)
    assert (nn_conv.stats['launches'], nn_conv.stats['applies']) == (launches, applies)
