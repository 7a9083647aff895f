"""CPU-only checks of the bipartite NNConv (DESIGN 4.10): the fp64 oracle against the reference's own NNConv_old run on
the union graph (golden G12), the constructor with an int and a pair ``in_channels``, the new C symbols, and the plan
size validation that needs no device."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from tests import bipartite_oracle as O
from tests.helpers import DenseNetLike

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _g12():
    from oracle import golden
    return golden.load(os.path.join(ROOT, 'tests', 'golden', 'g12_bipartite_nnconv.npz'))


def _sd(g, pre):
    return {k[len(pre) + 3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith(pre + 'sd_')}


def test_oracle_matches_reference_on_the_union_graph():
    g = _g12()
    for i in range(int(g['n_cases'])):
        pre = 'c%d_' % i
        n_src, n_dst, rb = [int(v) for v in g[pre + 'case']]
        sd = _sd(g, pre)
        ws = [sd['nn.layers.%d.weight' % j] for j in (0, 2, 4)]
        bs = [sd['nn.layers.%d.bias' % j] for j in (0, 2, 4)]
        out = O.bipartite_forward(torch.from_numpy(g[pre + 'x_src']), torch.from_numpy(g[pre + 'x_dst']),
                                  torch.from_numpy(g[pre + 'edge_index']), torch.from_numpy(g[pre + 'edge_attr']), ws, bs,
                                  sd.get('root'), sd.get('bias'), str(g[pre + 'aggr']), n_dst)
        ref = torch.from_numpy(g[pre + 'out']).double()
        assert out.shape == (n_dst, ref.size(1))
        assert float((out - ref).abs().max()) <= 1e-5 * max(1.0, float(ref.abs().max())), i
        assert ('root' in sd) == bool(rb)


def test_oracle_max_gives_zero_to_targets_without_in_edges():
    ei = torch.tensor([[0, 1, 1], [1, 1, 2]])
    ws, bs = [torch.ones(2, 1)], [torch.zeros(2)]
    out = O.bipartite_forward(torch.tensor([[1.0], [3.0]]), None, ei, torch.tensor([[1.0], [2.0], [-1.0]]), ws, bs,
                              None, None, 'max', 4)
    assert out[:, 0].tolist() == [0.0, 6.0, -3.0, 0.0]


def _conv(in_channels, out_channels=5, **kw):
    from graph_pde_b200.nn_conv import NNConv_old
    in_src = in_channels[0] if isinstance(in_channels, (tuple, list)) else in_channels
    return NNConv_old(in_channels, out_channels, DenseNetLike([3, 8, in_src * out_channels]), **kw)


def test_int_in_channels_keeps_shapes_keys_init_and_repr():
    torch.manual_seed(3)
    a = _conv(4)
    torch.manual_seed(3)
    b = _conv((4, 4))
    assert a.root.shape == (4, 5) and repr(a) == 'NNConv_old(4, 5)'
    assert list(a.state_dict()) == list(b.state_dict())
    for k, v in a.state_dict().items():            # the same draws: (4, 4) is the int's rule
        assert torch.equal(v, b.state_dict()[k]), k


def test_pair_in_channels_root_shape_init_bound_and_repr():
    torch.manual_seed(0)
    c = _conv((9, 2), 7)
    assert c.in_channels == (9, 2)
    assert c.root.shape == (2, 7) and c.bias.shape == (7,)
    assert repr(c) == 'NNConv_old((9, 2), 7)'
    assert list(c.state_dict()) == ['root', 'bias', 'nn.layers.0.weight', 'nn.layers.0.bias', 'nn.layers.2.weight',
                                    'nn.layers.2.bias']
    assert c.nn.layers[-1].out_features == 9 * 7
    bound = 1.0 / math.sqrt(9)                     # in_src, the message side
    big = _conv((9, 2), 300)
    for t in (big.root.detach(), big.bias.detach()):
        assert float(t.abs().max()) <= bound
        assert float(t.abs().max()) > 0.9 * bound  # 900 / 300 draws: the bound is the message side's, not 1/sqrt(2)
    c2 = _conv([9, 2], 7)
    assert c2.in_channels == (9, 2)


def test_new_symbols_are_declared_and_exported():
    from graph_pde_b200 import _lib
    names = ['nnconv_plan_sizes_bipartite', 'nnconv_plan_create_bipartite', 'nnconv_root_term',
             'nnconv_root_term_backward']
    header = open(os.path.join(ROOT, 'include', 'nnconv_b200.h')).read()
    for n in names:
        assert n in _lib.SYMBOLS and n + '(' in header
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    L = _lib.lib()
    for n in names:
        assert getattr(L, n) is not None


@pytest.mark.parametrize('n_src,n_dst,word', [(0, 5, 'n_src'), (5, 0, 'n_dst'), (-2, 3, 'n_src'), (4, -1, 'n_dst')])
def test_plan_sizes_reject_an_empty_side(n_src, n_dst, word):
    from graph_pde_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    L = _lib.lib()
    ws, tmp = ctypes.c_size_t(), ctypes.c_size_t()
    assert L.nnconv_plan_sizes_bipartite(100, n_src, n_dst, ctypes.byref(ws), ctypes.byref(tmp)) != 0
    msg = L.nnconv_last_error().decode()
    assert word + ' >= 1' in msg


def test_plan_sizes_grow_with_each_side():
    from graph_pde_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    L = _lib.lib()

    def sizes(e, a, b):
        ws, tmp = ctypes.c_size_t(), ctypes.c_size_t()
        assert L.nnconv_plan_sizes_bipartite(e, a, b, ctypes.byref(ws), ctypes.byref(tmp)) == 0
        return ws.value, tmp.value
    sq, sq_tmp = ctypes.c_size_t(), ctypes.c_size_t()
    assert L.nnconv_plan_sizes(1000, 50, ctypes.byref(sq), ctypes.byref(sq_tmp)) == 0
    assert sizes(1000, 50, 50) == (sq.value, sq_tmp.value)
    assert sizes(1000, 50, 5000)[0] > sizes(1000, 50, 50)[0]      # inv_deg over the targets
    assert sizes(1000, 5000, 50)[1] > sizes(1000, 50, 50)[1]      # per-source scratch


def test_host_refusals_need_no_device():
    c = _conv((3, 2), 4, flow='target_to_source')
    with pytest.raises(ValueError, match='target_to_source'):
        c((torch.zeros(5, 3), torch.zeros(4, 2)), torch.zeros(2, 1, dtype=torch.long), torch.zeros(1, 3))
    c = _conv((3, 2), 4)
    with pytest.raises(ValueError, match='size'):
        c((torch.zeros(5, 3), None), torch.zeros(2, 1, dtype=torch.long), torch.zeros(1, 3))
    with pytest.raises(ValueError, match='disagrees'):
        c((torch.zeros(5, 3), torch.zeros(4, 2)), torch.zeros(2, 1, dtype=torch.long), torch.zeros(1, 3), size=(6, 4))
    with pytest.raises(ValueError, match='disagrees'):
        c((torch.zeros(5, 3), torch.zeros(4, 2)), torch.zeros(2, 1, dtype=torch.long), torch.zeros(1, 3), size=(5, 3))
    c = _conv(4, 4)
    with pytest.raises(ValueError, match='one node set'):
        with torch.no_grad():
            c.residual_step((torch.zeros(5, 4), torch.zeros(4, 4)), torch.zeros(2, 1, dtype=torch.long),
                            torch.zeros(1, 3))
    with pytest.raises(ValueError, match='disagrees'):
        c(torch.zeros(5, 4), torch.zeros(2, 1, dtype=torch.long), torch.zeros(1, 3), size=(5, 6))


def test_golden_holds_data_only():
    g = _g12()
    for k in g.files:
        assert np.asarray(g[k]).dtype.kind in 'fiuU', k
