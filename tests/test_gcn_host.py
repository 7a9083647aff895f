"""CPU-only checks of GCNConv: the fp64 oracle against hand-computed outputs and the g9 fixture, the module API, the
drop-in import and the lattice builder."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import golden
from tests import gcn_oracle as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dense(edge_index, n, **kw):
    """A_hat as a dense matrix, through the oracle (x = I, W = I)."""
    return G.gcn_forward(torch.eye(n, dtype=torch.float64), edge_index, torch.eye(n, dtype=torch.float64), **kw)


def test_oracle_hand_computed_cases():
    # 0 -> 1, 0 -> 1 (duplicate), 2 -> 1, 1 -> 1 (a caller's loop), 2 -> 0 (asymmetric); node 3 isolated
    ei = torch.tensor([[0, 0, 2, 1, 2], [1, 1, 1, 1, 0]])
    A = _dense(ei, 4)
    # in-degrees without loops: 0: 1, 1: 3, 2: 0, 3: 0; one loop each (node 1 keeps its own, weight 1)
    deg = torch.tensor([2.0, 4.0, 1.0, 1.0], dtype=torch.float64)
    d = deg.pow(-0.5)
    want = torch.zeros(4, 4, dtype=torch.float64)
    want[1, 0] = 2 * d[0] * d[1]
    want[1, 2] = d[2] * d[1]
    want[0, 2] = d[2] * d[0]
    for i in range(4):
        want[i, i] = d[i] * d[i]
    # out = A_hat x: row = target, column = source
    assert torch.allclose(A, want)
    # improved: loops of weight 2 where the caller had none
    Ai = _dense(ei, 4, improved=True)
    degi = torch.tensor([3.0, 4.0, 2.0, 2.0], dtype=torch.float64)
    di = degi.pow(-0.5)
    assert math.isclose(Ai[0, 0].item(), 2 * di[0].item() ** 2)
    assert math.isclose(Ai[1, 1].item(), di[1].item() ** 2)        # the caller's loop keeps weight 1
    assert math.isclose(Ai[1, 0].item(), 2 * di[0].item() * di[1].item())
    # normalize=False: the plain sum over the caller's list, its loop included
    An = _dense(ei, 4, normalize=False)
    wantn = torch.zeros(4, 4, dtype=torch.float64)
    wantn[1, 0], wantn[1, 2], wantn[1, 1], wantn[0, 2] = 2, 1, 1, 1
    assert torch.equal(An, wantn)
    # add_self_loops=False: the caller's loop counts as an edge, nobody else gets one; isolated degree 0 -> 0
    Al = _dense(ei, 4, add_self_loops=False)
    dl = torch.tensor([1.0, 4.0, 0.0, 0.0], dtype=torch.float64)
    dli = torch.where(dl > 0, dl.pow(-0.5), torch.zeros_like(dl))
    assert math.isclose(Al[1, 1].item(), dli[1].item() ** 2)
    assert Al[2, 2].item() == 0 and Al[3, 3].item() == 0
    assert math.isclose(Al[1, 0].item(), 2 * dli[0].item() * dli[1].item())
    # degrees at the target: 2 -> 0 uses deg(0) = 1 + loop, not 0's out-degree
    assert math.isclose(A[0, 2].item(), d[2].item() * d[0].item())


def test_oracle_flow_swaps_rows():
    ei = torch.tensor([[0, 2, 3], [1, 1, 0]])
    a = _dense(ei, 4, flow='target_to_source')
    b = _dense(ei.flip(0), 4)
    assert torch.equal(a, b)


def test_oracle_gcn_net_matches_g9():
    from graph_pde_b200.models import GCN_Net
    rec = golden.load(os.path.join(ROOT, 'tests', 'golden', 'g9_gcn_net.npz'))
    torch.manual_seed(90)
    net = GCN_Net(32, 16, 2, in_width=1)
    sd = net.state_dict()
    assert list(sd.keys()) == list(rec['keys'])
    for k, v in sd.items():       # the reference's init stream, value for value
        assert np.array_equal(v.double().numpy(), rec['sd_' + k]), k
    # the oracle through the same wiring reproduces the fixture
    ref = G.GCNConv
    ei = torch.from_numpy(rec['edge_index'])
    x = torch.from_numpy(rec['x'])
    p = {k: torch.from_numpy(rec['sd_' + k]) for k in rec['keys']}
    h = x @ p['fc_in.weight'].t() + p['fc_in.bias']
    for _ in range(2):
        for c in ('conv1', 'conv2', 'conv3', 'conv4'):
            h = torch.relu(G.gcn_forward(h, ei, p[c + '.weight'], p[c + '.bias']))
    h = torch.relu(h @ p['fc_out1.weight'].t() + p['fc_out1.bias'])
    out = h @ p['fc_out2.weight'].t() + p['fc_out2.bias']
    assert torch.allclose(out, torch.from_numpy(rec['out']), rtol=1e-12, atol=1e-12)
    assert repr(ref(128, 128)) == 'GCNConv(128, 128)'


def test_module_api():
    from graph_pde_b200 import GCNConv
    conv = GCNConv(128, 64)
    assert repr(conv) == 'GCNConv(128, 64)'
    assert [(k, tuple(v.shape)) for k, v in conv.state_dict().items()] == [('weight', (128, 64)), ('bias', (64,))]
    assert GCNConv(16, 16, bias=False).bias is None
    torch.manual_seed(0)
    conv = GCNConv(128, 128)
    stdv = math.sqrt(6.0 / 256)
    w = conv.weight.detach()
    assert w.abs().max().item() <= stdv and w.abs().max().item() > 0.95 * stdv
    assert abs(w.mean().item()) < 0.01 and abs(w.var().item() - stdv ** 2 / 3) < 0.1 * stdv ** 2 / 3
    assert torch.equal(conv.bias.detach(), torch.zeros(128))
    # the same stream as the oracle's PyG 1.x module
    torch.manual_seed(5)
    a = GCNConv(32, 48)
    torch.manual_seed(5)
    b = G.GCNConv(32, 48)
    assert torch.equal(a.weight, b.weight) and torch.equal(a.bias, b.bias)
    # PyG 2.x checkpoints keep W as lin.weight [out, in]
    W = torch.randn(48, 32)
    a.load_state_dict({'lin.weight': W, 'bias': torch.ones(48)})
    assert torch.equal(a.weight.detach(), W.t()) and torch.equal(a.bias.detach(), torch.ones(48))
    a.load_state_dict(b.state_dict())
    assert torch.equal(a.weight, b.weight)
    with pytest.raises(NotImplementedError, match='edge_weight'):
        a(torch.zeros(3, 32), torch.zeros(2, 0, dtype=torch.long), torch.ones(0))
    with pytest.raises(TypeError):
        GCNConv(16, 16, bogus=1)
    GCNConv(16, 16, improved=True, cached=True, add_self_loops=False, normalize=False, precision='fp32',
            flow='target_to_source')


def test_dropin_import_resolves():
    code = ('import sys; from torch_geometric.nn import GCNConv, NNConv; '
            'import graph_pde_b200.gcn as g, graph_pde_b200.nn_conv as n; '
            'assert GCNConv is g.GCNConv and NNConv is n.NNConv; print("ok")')
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, 'dropin'), ROOT]))
    res = subprocess.run([sys.executable, '-c', code], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True, cwd=ROOT)
    assert res.returncode == 0 and 'ok' in res.stdout, res.stdout


def test_grid_edge_3x2():
    from graph_pde_b200.graphs import grid_edge
    grid, ei = grid_edge(3, 2)
    # node i = y * 3 + x; per node: right pair unless last column, then up pair unless last row
    want = [(0, 1), (1, 0), (0, 3), (3, 0),
            (1, 2), (2, 1), (1, 4), (4, 1),
            (2, 5), (5, 2),
            (3, 4), (4, 3),
            (4, 5), (5, 4)]
    assert [tuple(p) for p in ei.t().tolist()] == want
    assert ei.dtype == torch.int64
    assert torch.allclose(grid, torch.tensor([[0, 0], [0.5, 0], [1, 0], [0, 1], [0.5, 1], [1, 1]], dtype=torch.float32))


@pytest.mark.parametrize('n,amp,seed,loops', [(2000, 3, 0, 50), (421 * 421, 1, 7, 0)])
def test_exact_probe_budget(n, amp, seed, loops):
    """The exact probes of test_gpu_gcn.py are exact on every path: every norm is a power of two; each row of z = A_hat x
    and w = A_hat^T g, in units of its smallest norm (1/16), has at most 8 significant bits (bf16 keeps them after the
    power-of-two row scaling); and the fp32 sums of out, dW and db stay below 2^24 units whatever their order."""
    from tests.test_gpu_gcn import _pow4_graph
    ei = _pow4_graph(n, seed=seed, loops=loops)
    src, dst, norm = G.gcn_norm(ei, n)
    m, e = np.frexp(norm.numpy())
    assert np.all(m == 0.5) and norm.min().item() >= 1 / 16
    absA = torch.zeros(n, dtype=torch.float64).index_add_(0, dst, norm)        # sum_m |A_hat[n, m]| (row sums)
    absAT = torch.zeros(n, dtype=torch.float64).index_add_(0, src, norm)       # column sums: w = A_hat^T g
    z_units = (absA * amp * 16).max().item()
    w_units = (absAT * amp * 16).max().item()
    assert z_units <= 256 and w_units <= 256, (z_units, w_units)
    assert 128 * z_units * 2 < 2 ** 24                                            # out: 128 terms of |z| |W| <= 2
    assert n * amp * w_units < 2 ** 24                                            # dW = x^T w over all rows
