"""GCNConv on the GPU: parity with the fp64 oracle at every precision, the kernel each shape runs, gradients, exact
integer probes up to the 421^2 lattice, range safety, run-to-run bit equality, CUDA-graph capture and the empty graph."""
import os

import numpy as np
import pytest
import torch

from oracle import golden
from tests import gcn_oracle as G
from tests.helpers import TOL, rel_err

pytestmark = pytest.mark.gpu
DEV = 'cuda'
PRECS = ('f16', 'bf16', 'f16x2', 'fp32')
GRAD_TOL = {'f16': 3e-3, 'bf16': 3e-2, 'f16x2': 1e-4, 'fp32': 2e-5}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _conv(cin, cout, precision, seed=0, **kw):
    from graph_pde_b200 import GCNConv
    torch.manual_seed(seed)
    conv = GCNConv(cin, cout, precision=precision, **kw).to(DEV)
    with torch.no_grad():
        conv.bias.uniform_(-0.5, 0.5) if conv.bias is not None else None
    return conv


def _messy_graph(n=700, e=5000, seed=1):
    """Hub sources and targets, duplicate edges, caller self loops and isolated nodes."""
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n - 20, (e,), generator=g)
    dst = torch.randint(0, n - 20, (e,), generator=g)
    src[:400] = 3                      # hub source
    dst[400:700] = 5                   # hub target
    src[700:720], dst[700:720] = src[0], dst[0]        # duplicates
    dst[720:760] = src[720:760]        # self loops
    return torch.stack([src, dst]).to(DEV), n          # nodes n-20 .. n-1: isolated


def _ref(conv, x, ei, **kw):
    return G.gcn_forward(x.double(), ei, conv.weight.detach().double(),
                         None if conv.bias is None else conv.bias.detach().double(),
                         improved=conv.improved, add_self_loops=conv.add_self_loops, normalize=conv.normalize,
                         flow=conv.flow)


@pytest.mark.parametrize('precision', PRECS)
@pytest.mark.parametrize('cin,cout', [(16, 16), (64, 64), (128, 128), (48, 80)])
def test_parity_messy_graph(precision, cin, cout):
    ei, n = _messy_graph()
    conv = _conv(cin, cout, precision)
    x = torch.randn(n, cin, device=DEV)
    with torch.no_grad():
        out = conv(x, ei)
    assert rel_err(out, _ref(conv, x, ei)) < TOL[precision], precision


@pytest.mark.parametrize('precision', PRECS)
@pytest.mark.parametrize('kw', [dict(improved=True), dict(add_self_loops=False), dict(normalize=False),
                                dict(flow='target_to_source'), dict(bias=False)])
def test_parity_options(precision, kw):
    ei, n = _messy_graph(seed=2)
    conv = _conv(64, 32, precision, **kw)
    x = torch.randn(n, 64, device=DEV)
    with torch.no_grad():
        out = conv(x, ei)
    assert rel_err(out, _ref(conv, x, ei)) < TOL[precision], (precision, kw)


@pytest.mark.parametrize('precision', PRECS)
def test_gcn_net_on_g9(precision):
    from graph_pde_b200.models import GCN_Net
    rec = golden.load(os.path.join(ROOT, 'tests', 'golden', 'g9_gcn_net.npz'))
    torch.manual_seed(90)
    net = GCN_Net(32, 16, 2, in_width=1, precision=precision).to(DEV)

    class D(object):
        pass
    d = D()
    d.x = torch.from_numpy(rec['x']).float().to(DEV)
    d.edge_index = torch.from_numpy(rec['edge_index']).to(DEV)
    with torch.no_grad():
        out = net(d)
    assert rel_err(out, torch.from_numpy(rec['out'])) < 4 * TOL[precision], precision


_NAMES_SCRIPT = """
import sys, time, torch
sys.path.insert(0, %r)
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile
from graph_pde_b200 import GCNConv
from tests.test_gpu_gcn import _messy_graph
precision, cin, cout = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
ei, n = _messy_graph()
conv = GCNConv(cin, cout, precision=precision).cuda()
x = torch.randn(n, cin, device='cuda', requires_grad=True)
try:
    conv(x, ei).square().sum().backward()
except Exception as e:
    print('ERROR', type(e).__name__, e)
    sys.exit(0)
torch.cuda.synchronize()
for _ in range(4):
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        conv(x, ei).square().sum().backward()
        torch.cuda.synchronize()
        time.sleep(0.02)
    names = {e.name for e in prof.events() if e.device_type == DeviceType.CUDA}
    if names:
        break
print('NAMES', ' '.join(sorted(names)))
""" % ROOT


def _kernel_names(precision, cin, cout):
    """Kernels one forward + backward launches, profiled in a fresh process (the profiler state of the test process is
    left alone); 'ERROR ...' if the call raised."""
    import subprocess
    import sys
    res = subprocess.run([sys.executable, '-c', _NAMES_SCRIPT, precision, str(cin), str(cout)], cwd=ROOT,
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert res.returncode == 0, res.stdout
    return res.stdout


@pytest.mark.parametrize('precision', ('f16', 'bf16', 'f16x2'))
def test_reference_shape_runs_the_fused_kernel(precision):
    names = _kernel_names(precision, 128, 128)
    assert 'NAMES' in names and 'k_gcn_tc' in names, names
    assert 'k_gcn_gather' not in names and 'k_sgemm_nt' not in names, names


def test_fp32_and_wide_shapes_run_the_cuda_cores():
    for precision, cout in (('fp32', 128), ('fp32', 144)):
        names = _kernel_names(precision, 128, cout)
        assert 'NAMES' in names and 'k_gcn_gather' in names and 'k_sgemm_nt' in names, names
        assert 'k_gcn_tc' not in names, names
        ei, n = _messy_graph()
        conv = _conv(128, cout, precision)
        x = torch.randn(n, 128, device=DEV)
        with torch.no_grad():
            assert rel_err(conv(x, ei), _ref(conv, x, ei)) < TOL['fp32']
    names = _kernel_names('f16', 128, 144)
    assert 'ERROR NNConvLibraryError' in names and "'fp32'" in names, names


OPTIONS = [dict(improved=True), dict(add_self_loops=False), dict(normalize=False), dict(flow='target_to_source'),
           dict(bias=False)]


def _check_gradients(precision, cin, cout, **kw):
    ei, n = _messy_graph(seed=3)
    conv = _conv(cin, cout, precision, **kw)
    x = torch.randn(n, cin, device=DEV, requires_grad=True)
    gout = torch.randn(n, cout, device=DEV)
    (conv(x, ei) * gout).sum().backward()
    x64 = x.detach().double().requires_grad_()
    w64 = conv.weight.detach().double().requires_grad_()
    b64 = None if conv.bias is None else conv.bias.detach().double().requires_grad_()
    ref = G.gcn_forward(x64, ei, w64, b64, improved=conv.improved, add_self_loops=conv.add_self_loops,
                        normalize=conv.normalize, flow=conv.flow)
    (ref * gout.double()).sum().backward()
    errs = {'x': rel_err(x.grad, x64.grad), 'weight': rel_err(conv.weight.grad, w64.grad)}
    if b64 is not None:
        errs['bias'] = rel_err(conv.bias.grad, b64.grad)
    print('gcn grad err', precision, cin, cout, kw, errs)
    assert max(errs.values()) < GRAD_TOL[precision], (precision, kw, errs)


@pytest.mark.parametrize('precision', PRECS)
@pytest.mark.parametrize('cin,cout', [(128, 128), (32, 96)])
def test_gradients(precision, cin, cout):
    _check_gradients(precision, cin, cout)


@pytest.mark.parametrize('precision', PRECS)
@pytest.mark.parametrize('kw', OPTIONS)
def test_gradients_options(precision, kw):
    """The backward of every normalisation option and flow: the by-source CSR and the per-node diagonal they build."""
    _check_gradients(precision, 64, 32, **kw)


def test_edge_index_is_checked():
    from graph_pde_b200 import gcn
    ei, n = _messy_graph()
    conv = _conv(32, 32, 'f16')
    x = torch.randn(n, 32, device=DEV)
    for bad in (ei.int(), ei.t().contiguous(), ei[0], ei.float()):
        with pytest.raises(ValueError, match='edge_index'):
            conv(x, bad)
    with pytest.raises(RuntimeError, match='edge_index'):
        conv(x, ei.cpu())
    # the graphs are cached per edge_index and dropped by clear_caches
    from graph_pde_b200.nn_conv import clear_caches
    clear_caches()
    before = gcn.stats['graphs_built']
    with torch.no_grad():
        conv(x, ei)
        conv(x, ei)
    assert gcn.stats['graphs_built'] == before + 1 and len(gcn._GRAPH_CACHE) == 1
    clear_caches()
    assert len(gcn._GRAPH_CACHE) == 0
    with torch.no_grad():
        conv(x, ei)
    assert gcn.stats['graphs_built'] == before + 2


def _pow4_graph(n, degs=(3, 15), seed=0, loops=0):
    """Every node's in-degree (without loops) is 3 or 15, so deg = 4 or 16 with its loop: every norm is a power of two.
    ``loops`` nodes of in-degree 3 also carry a caller self loop (weight 1, the same as the added one)."""
    g = torch.Generator().manual_seed(seed)
    d = torch.tensor(degs)[torch.randint(0, len(degs), (n,), generator=g)]
    dst = torch.repeat_interleave(torch.arange(n), d)
    src = torch.randint(0, n - 1, (dst.numel(),), generator=g)
    src = src + (src >= dst).long()            # never a loop
    perm = torch.randperm(dst.numel(), generator=g)
    src, dst = src[perm], dst[perm]
    if loops:
        ln = torch.nonzero(d == degs[0]).flatten()[:loops]
        src, dst = torch.cat([src, ln]), torch.cat([dst, ln])
    return torch.stack([src, dst])


def _exact_probe(n, precision, cin=128, cout=128, amp=3, seed=0, loops=0):
    ei = _pow4_graph(n, seed=seed, loops=loops).to(DEV)
    g = torch.Generator().manual_seed(seed + 1)
    conv = _conv(cin, cout, precision)
    with torch.no_grad():
        conv.weight.copy_(torch.randint(-2, 3, (cin, cout), generator=g).float())
        conv.bias.copy_(torch.randint(-4, 5, (cout,), generator=g).float())
    x = torch.randint(-amp, amp + 1, (n, cin), generator=g).float().to(DEV).requires_grad_()
    gout = torch.randint(-amp, amp + 1, (n, cout), generator=g).float().to(DEV)
    out = conv(x, ei)
    out.backward(gout)
    x64 = x.detach().double().requires_grad_()
    w64 = conv.weight.detach().double().requires_grad_()
    b64 = conv.bias.detach().double().requires_grad_()
    ref = G.gcn_forward(x64, ei, w64, b64)
    ref.backward(gout.double())
    return [(name, a.double(), b.detach()) for name, a, b in
            (('out', out, ref), ('dx', x.grad, x64.grad), ('dW', conv.weight.grad, w64.grad),
             ('db', conv.bias.grad, b64.grad))]


@pytest.mark.parametrize('precision', PRECS)
def test_exact_probe_small(precision):
    for name, got, want in _exact_probe(2000, precision, loops=50):
        bad = (got != want).any(dim=-1).nonzero().flatten()[:5].tolist() if got.dim() > 1 else []
        assert torch.equal(got, want), (precision, name, bad)


@pytest.mark.parametrize('precision', PRECS)
def test_exact_probe_421(precision):
    """N = 421^2 with in-degrees 3 and 15: one lost or misrouted edge changes some node's output."""
    for name, got, want in _exact_probe(421 * 421, precision, amp=1, seed=7):
        assert torch.equal(got, want), (precision, name)


@pytest.mark.parametrize('precision', PRECS)
@pytest.mark.parametrize('e', (-20, 20))
def test_range_safety(precision, e):
    ei, n = _messy_graph(seed=4)
    conv = _conv(64, 64, precision, bias=False)
    x = torch.randn(n, 64, device=DEV) * 2.0 ** e
    with torch.no_grad():
        out = conv(x, ei)
        assert bool(torch.isfinite(out).all())
        assert rel_err(out, _ref(conv, x, ei)) < TOL[precision], (precision, e)


@pytest.mark.parametrize('precision', PRECS)
def test_bitwise_reproducible(precision):
    ei, n = _messy_graph(seed=5)
    conv = _conv(128, 128, precision)
    x = torch.randn(n, 128, device=DEV, requires_grad=True)
    gout = torch.randn(n, 128, device=DEV)
    runs = []
    for _ in range(2):
        x.grad, conv.weight.grad, conv.bias.grad = None, None, None
        out = conv(x, ei)
        out.backward(gout)
        runs.append([out.detach().clone(), x.grad.clone(), conv.weight.grad.clone(), conv.bias.grad.clone()])
    for a, b in zip(*runs):
        assert torch.equal(a, b), precision


@pytest.mark.parametrize('precision', ('f16', 'f16x2', 'fp32'))
def test_empty_graph_is_self_loops_only(precision):
    conv = _conv(32, 32, precision)
    x = torch.randn(50, 32, device=DEV)
    ei = torch.zeros(2, 0, dtype=torch.long, device=DEV)
    with torch.no_grad():
        out = conv(x, ei)
    want = x @ conv.weight + conv.bias
    assert rel_err(out, want) < TOL[precision]


@pytest.mark.parametrize('precision', ('f16', 'f16x2'))
def test_graphed_train_step_matches_eager(precision):
    import torch.nn.functional as F
    from graph_pde_b200 import GraphedTrainStep
    from graph_pde_b200.graphs import grid_edge
    from graph_pde_b200.models import GCN_Net
    grid, ei = grid_edge(85, 85, device=DEV)

    class D(object):
        pass

    def make():
        torch.manual_seed(3)
        m = GCN_Net(64, 32, 2, in_width=2, precision=precision).to(DEV)
        return m, torch.optim.Adam(m.parameters(), lr=1e-3, capturable=True)
    y = torch.randn(grid.size(0), 1, device=DEV)
    model_e, opt_e = make()
    model_g, opt_g = make()
    d = D()
    d.x, d.edge_index = grid, ei
    step = GraphedTrainStep(lambda xx, yy: F.mse_loss(model_g(d), yy), model_g, opt_g, grid, y)
    for i in range(3):
        opt_e.zero_grad(set_to_none=True)
        loss_e = F.mse_loss(model_e(d), y)
        loss_e.backward()
        opt_e.step()
        loss_g = step.replay()
        assert rel_err(loss_g, loss_e.detach()) < 1e-5, (precision, i)
        for (name, pg), pe in zip(model_g.named_parameters(), model_e.parameters()):
            assert rel_err(pg, pe) < 1e-5, (precision, i, name)


@pytest.mark.parametrize('precision', PRECS)
def test_full_lattice_gcn_stack(precision):
    """neurips4_GCN.py's configuration: 421^2 grid_edge lattice, width 128, four convs applied 4 times (16 applications),
    against the oracle's ops in fp32 on the GPU."""
    from graph_pde_b200.graphs import grid_edge
    _, ei = grid_edge(421, 421, device=DEV)
    n = 421 * 421
    convs = [_conv(128, 128, precision, seed=10 + i) for i in range(4)]
    x0 = torch.randn(n, 128, device=DEV)
    src, dst, norm = G.gcn_norm(ei, n, dtype=torch.float32)
    with torch.no_grad():
        x, r = x0, x0
        for _ in range(4):
            for c in convs:
                x = torch.relu(c(x, ei))
                xw = r @ c.weight
                r = torch.relu(torch.zeros_like(xw).index_add_(0, dst, norm[:, None] * xw[src]) + c.bias)
    assert rel_err(x, r) < 4 * TOL[precision], (precision, rel_err(x, r))


def test_graphed_forward_replays_gcn_net():
    from graph_pde_b200 import GraphedForward
    from graph_pde_b200.graphs import grid_edge
    from graph_pde_b200.models import GCN_Net
    grid, ei = grid_edge(85, 85, device=DEV)

    class D(object):
        pass
    d = D()
    d.x, d.edge_index = grid.clone(), ei
    torch.manual_seed(4)
    model = GCN_Net(64, 32, 2, in_width=2).to(DEV)
    g = GraphedForward(model, d)
    d.x.copy_(torch.rand_like(grid))
    with torch.no_grad():
        want = model(d)
    assert torch.equal(g.replay(), want)
