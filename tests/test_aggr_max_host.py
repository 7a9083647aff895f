"""aggr='max' on the CPU: the fp64 reference of tests/max_oracle.py against the PyG stub's scatter_reduce, its tie, -0
and NaN rules, its gradients, and the exactness of the probes the GPU tests run with max.

Why an add-exact probe is exact for max: tests/probes.assert_exact proves that every message m_e and every fp32 sum
of aggr='add' stays within 2^22 quanta.  Max adds no sum across edges at a target: it selects one message (a value the
add proof already covers) and adds it once to the node's root / bias term, a sum of |terms| no larger than add's.  In
the backward, max only replaces some of the gathered gradient entries G_e[o] = g[dst, o] by 0, so every source sum of
the add proof loses terms and none grows.  So each probe's add proof is also its max proof.
"""
import importlib.util
import os

import pytest
import torch

from oracle import nnconv_oracle as O
from tests import max_oracle as M
from tests import probes as P

_STUB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle', 'pyg_stub', 'torch_geometric',
                     'nn', 'conv', '__init__.py')


def _stub_message_passing():
    spec = importlib.util.spec_from_file_location('_pyg_stub_conv', _STUB)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.MessagePassing


def _random_case(seed, n=40, e=300, cin=3, cout=5, k_in=4):
    g = torch.Generator().manual_seed(seed)
    ei = torch.stack([torch.randint(0, n, (e,), generator=g), torch.randint(0, n - 5, (e,), generator=g)])
    x = torch.randn(n, cin, generator=g, dtype=torch.float64)
    ea = torch.randn(e, k_in, generator=g, dtype=torch.float64)
    ws = [torch.randn(16, k_in, generator=g, dtype=torch.float64), torch.randn(cin * cout, 16, generator=g,
                                                                               dtype=torch.float64)]
    bs = [torch.randn(16, generator=g, dtype=torch.float64), torch.randn(cin * cout, generator=g, dtype=torch.float64)]
    root = torch.randn(cin, cout, generator=g, dtype=torch.float64)
    bias = torch.randn(cout, generator=g, dtype=torch.float64)
    return ei, x, ea, ws, bs, root, bias


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_max_matches_pyg_scatter_reduce(seed):
    """The three-step oracle equals the stub MessagePassing's scatter_reduce('amax', include_self=False) on zeros,
    root and bias added as NNConv_old.update does; nodes 35..39 have no in-edges and get the root / bias term only."""
    ei, x, ea, ws, bs, root, bias = _random_case(seed)
    cin, cout = root.shape

    class StubConv(_stub_message_passing()):
        def __init__(self):
            super().__init__(aggr='max')

        def forward(self, x):
            return self.propagate(ei, x=x, pseudo=ea)

        def message(self, x_j, pseudo):
            k = O.dense_net(pseudo, ws, bs).view(-1, cin, cout)
            return torch.matmul(x_j.unsqueeze(1), k).squeeze(1)

        def update(self, aggr_out, x):
            return aggr_out + x @ root + bias

    ref = StubConv()(x)
    out, am = M.nnconv_forward_max(x, ei, ea, ws, bs, root, bias)
    assert torch.equal(out, ref)
    assert bool((am[35:] == -1).all())
    assert bool((am[:35] >= 0).all())


def test_tie_rule_zero_sign_and_nan():
    """Duplicate edges tie and the smallest caller index wins, whatever order the edges come in; -0 ties with +0;
    a NaN message wins and among NaN messages the smallest index wins; an empty node is 0 with argmax -1."""
    dst = torch.tensor([0, 0, 0, 1, 1, 1, 2, 2, 2, 3])
    msg = torch.tensor([[1., -0.0, 5.], [3., 0.0, float('nan')], [3., -1., float('nan')],   # node 0
                        [2., 2., -7.], [2., 2., -7.], [1., 2., -8.],                           # node 1: duplicates
                        [-0.0, float('nan'), 1.], [0.0, 4., 1.], [-3., float('nan'), 1.],       # node 2
                        [9., 9., 9.]], dtype=torch.float64)
    am = M.winners(msg, dst, 5)
    assert am[0].tolist() == [1, 0, 1]
    assert am[1].tolist() == [3, 3, 3]
    assert am[2].tolist() == [6, 6, 6]
    assert am[3].tolist() == [9, 9, 9]
    assert am[4].tolist() == [-1, -1, -1]
    term = M.max_term(msg, am)
    assert torch.isnan(term[0, 2]) and torch.isnan(term[2, 1])
    assert term[4].tolist() == [0., 0., 0.]
    # the same edges in reverse order: the winners are the same edges (now at mirrored caller indices)
    rev = torch.arange(msg.size(0) - 1, -1, -1)
    am_r = M.winners(msg[rev], dst[rev], 5)
    e = msg.size(0)
    for n in range(4):
        for o in range(3):
            # among tied edges the reversed list picks the one that was LAST before, so compare the values instead
            a, b = int(am[n, o]), int(e - 1 - am_r[n, o])
            va, vb = msg[a, o], msg[b, o]
            assert (bool(torch.isnan(va)) and bool(torch.isnan(vb))) or float(va) == float(vb)


def test_gradients_reach_only_the_winners():
    """fp64 autograd through the oracle: the gradient of out[n, o] reaches the winning message and no other; the
    message gradients of each node and channel sum to the output gradient."""
    ei, x, ea, ws, bs, root, bias = _random_case(3)
    cin, cout = root.shape
    src, dst = ei
    msg = M.messages(x, src, ea, ws, bs, cin, cout).detach().requires_grad_(True)
    am = M.winners(msg, dst, x.size(0))
    g = torch.randn(x.size(0), cout, dtype=torch.float64)
    (M.max_term(msg, am) * g).sum().backward()
    won = torch.zeros_like(msg, dtype=torch.bool)
    for n in range(x.size(0)):
        for o in range(cout):
            if am[n, o] >= 0:
                won[am[n, o], o] = True
    assert bool((msg.grad[~won] == 0).all())
    has_in = torch.bincount(dst, minlength=x.size(0)) > 0
    summed = torch.zeros(x.size(0), cout, dtype=torch.float64).index_add_(0, dst, msg.grad)
    assert torch.equal(summed[has_in], g[has_in])


@pytest.mark.parametrize('name,precision', [('mixed', 'f16'), ('mixed', 'f16x2'), ('mixed', 'fp32'),
                                            ('partial_tiles', 'bf16'), ('asymmetric_t2s', 'f16'), ('batch', 'f16'),
                                            ('nc16', 'f16'), ('out128', 'f16'), ('kp1088', 'f16')])
def test_forward_probes_are_exact_and_most_edges_win(name, precision):
    """The forward probes of tests/test_gpu_aggr_max.py pass assert_exact (the add proof, see the module docstring),
    and at least half of their edges win some (node, channel): a probe on which few edges can win would not notice
    a lost or misrouted loser."""
    p = P.probe(P.FORWARD, name, precision=precision)
    P.assert_exact(p, precision)
    src, dst = p.src_dst()
    msg = M.messages(p.x[0], src, p.ea.double(), p.ws, p.bs, p.cin, p.cout)
    am = M.winners(msg, dst, p.n_nodes)
    assert M.win_share(am, src.numel()) >= 0.5, (name, M.win_share(am, src.numel()))


@pytest.mark.parametrize('name,precision', [('mixed', 'f16'), ('mixed', 'f16x2'), ('cuda_core_out32', 'fp32'),
                                            ('cuda_core_in128', 'fp32'), ('asymmetric_t2s', 'f16')])
def test_backward_probes_are_exact(name, precision):
    P.assert_exact(P.probe(P.BACKWARD, name, precision=precision), precision)
