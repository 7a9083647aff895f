"""CPU-only checks of the bipartite DiagNNConv and GaussianNNConv (DESIGN 4.10): the fp64 restatement against the
reference's own NNConv and NNConv_Gaussian run on the union graph (golden G13), forward and gradients; the constructor
and its refusal of a pair ``in_channels``; and the ValueErrors of the pair / size checks, which need no device."""
import os

import numpy as np
import pytest
import torch

from tests import bipartite_channelwise_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _g13():
    from oracle import golden
    return golden.load(os.path.join(ROOT, 'tests', 'golden', 'g13_bipartite_channelwise.npz'))


def _close(a, ref, tol):
    ref = torch.as_tensor(ref).double()
    return float((a.detach() - ref).abs().max()) <= tol * max(1.0, float(ref.abs().max()))


def test_oracle_matches_reference_on_the_union_graph():
    g = _g13()
    kinds = set()
    for i in range(int(g['n_cases'])):
        pre = 'c%d_' % i
        kind, aggr, n_src, n_dst, rb = [str(v) for v in g[pre + 'case']]
        n_dst = int(n_dst)
        kinds.add((kind, aggr, rb))
        sd = {k[len(pre) + 3:]: torch.from_numpy(g[k]).double().requires_grad_() for k in g.files
              if k.startswith(pre + 'sd_')}
        xs = torch.from_numpy(g[pre + 'x_src']).double().requires_grad_()
        xd = torch.from_numpy(g[pre + 'x_dst']).double().requires_grad_()
        ea = torch.from_numpy(g[pre + 'edge_attr']).double().requires_grad_()
        if kind == 'diag':
            d = O.diag_d(ea, [sd['nn.0.weight'], sd['nn.2.weight']], [sd['nn.0.bias'], sd['nn.2.bias']])
        else:
            d = O.gauss_d(ea, torch.ones(1, dtype=torch.float64) @ sd['nn.weight'].t() + sd['nn.bias'])
        out, _ = O.forward(xs, xd, torch.from_numpy(g[pre + 'edge_index']), d, sd.get('root'), sd.get('bias'), aggr,
                           n_dst)
        assert out.shape == (n_dst, xs.size(1))
        assert _close(out, g[pre + 'out'], 1e-5), (i, kind, aggr)
        (out * torch.from_numpy(g[pre + 'gw']).double()).sum().backward()
        for name, t in [('x_src', xs), ('x_dst', xd), ('edge_attr', ea)] + list(sd.items()):
            grad = t.grad if t.grad is not None else torch.zeros_like(t)   # x_dst without root: no path, grad 0
            assert _close(grad, g[pre + 'grad_' + name], 1e-4), (i, kind, aggr, name)
        assert ('root' in sd) == (rb == 'True')
    assert {(k, a) for k, a, _ in kinds} == {(k, a) for k in ('diag', 'gauss') for a in ('add', 'mean', 'max')}


def test_oracle_gives_targets_without_in_edges_only_the_root_term():
    ei = torch.tensor([[0, 1, 1], [1, 1, 2]])
    d = torch.tensor([[1.0], [2.0], [-1.0]], dtype=torch.float64)
    xs = torch.tensor([[1.0], [3.0]], dtype=torch.float64)
    for aggr, col in (('add', [0.0, 7.0, -3.0, 0.0]), ('mean', [0.0, 3.5, -3.0, 0.0]), ('max', [0.0, 6.0, -3.0, 0.0])):
        out, _ = O.forward(xs, None, ei, d, None, None, aggr, 4)
        assert out[:, 0].tolist() == col, aggr


def _diag(in_channels=8, out_channels=8, **kw):
    from graph_pde_b200.nn_conv import DiagNNConv
    return DiagNNConv(in_channels, out_channels, torch.nn.Sequential(torch.nn.Linear(3, 16), torch.nn.ReLU(),
                                                                     torch.nn.Linear(16, out_channels)), **kw)


def _gauss(in_channels=8, out_channels=8, **kw):
    from graph_pde_b200.gauss import GaussianNNConv
    return GaussianNNConv(in_channels, out_channels, torch.nn.Linear(1, out_channels), **kw)


@pytest.mark.parametrize('make', [_diag, _gauss])
@pytest.mark.parametrize('root_weight', [True, False])
def test_pair_in_channels_raises_not_implemented(make, root_weight):
    for pair in ((8, 8), [8, 4]):
        with pytest.raises(NotImplementedError, match=r'in_channels \(8, %d\), out_channels 8' % pair[1]):
            make(pair, 8, root_weight=root_weight)


@pytest.mark.parametrize('make', [_diag, _gauss])
def test_int_in_channels_keeps_shapes_keys_and_repr(make):
    c = make(8, 8)
    name = type(c).__name__
    assert repr(c) == '%s(8, 8)' % name
    assert c.root.shape == (8, 8) and c.bias.shape == (8,)
    assert [k for k in c.state_dict() if not k.startswith('nn.')] == ['root', 'bias']


@pytest.mark.parametrize('make', [_diag, _gauss])
def test_value_errors_before_any_device_work(make):
    """CPU tensors: each refusal below is raised by the host checks, before the first CUDA call could fail."""
    ei, ea = torch.zeros(2, 1, dtype=torch.long), torch.ones(1, 3)
    xs, xd = torch.zeros(5, 8), torch.zeros(4, 8)
    c = make(flow='target_to_source')
    with pytest.raises(ValueError, match='target_to_source'):
        c((xs, xd), ei, ea)
    c = make()
    with pytest.raises(ValueError, match='size'):
        c((xs, None), ei, ea)
    with pytest.raises(ValueError, match=r'size\[0\] = 6 disagrees'):
        c((xs, xd), ei, ea, size=(6, 4))
    with pytest.raises(ValueError, match=r'size\[1\] = 3 disagrees'):
        c((xs, xd), ei, ea, size=(5, 3))
    with pytest.raises(ValueError, match='size must be'):
        c((xs, xd), ei, ea, size=(5, 4, 1))
    with pytest.raises(ValueError, match='at least one target'):
        c((xs, None), ei, ea, size=(5, 0))
    with pytest.raises(ValueError, match='pair'):
        c((xs, xd, xd), ei, ea)
    with pytest.raises(ValueError, match='one node set'):
        c(xs, ei, ea, size=(5, 6))


def test_dropin_classes_take_the_same_checks():
    import importlib.util
    spec = importlib.util.spec_from_file_location('dropin_nn_conv', os.path.join(ROOT, 'dropin', 'nn_conv.py'))
    dropin = importlib.util.module_from_spec(spec)       # not under the name nn_conv: no other test sees it
    spec.loader.exec_module(dropin)
    for cls, nn in ((dropin.NNConv, torch.nn.Linear(3, 8)), (dropin.NNConv_Gaussian, torch.nn.Linear(1, 8))):
        with pytest.raises(NotImplementedError, match='in_channels'):
            cls((8, 8), 8, nn)
        with pytest.raises(ValueError, match='disagrees'):
            cls(8, 8, nn)((torch.zeros(5, 8), torch.zeros(4, 8)), torch.zeros(2, 1, dtype=torch.long), torch.ones(1, 3),
                          size=(5, 3))


def test_golden_holds_data_only():
    g = _g13()
    for k in g.files:
        assert np.asarray(g[k]).dtype.kind in 'fiuU', k
