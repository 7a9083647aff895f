"""The diagonal-kernel NNConv on the CPU: the fp64 oracle against the reference's own outputs (g8), the module's init
stream, state-dict keys and repr, its shape refusal, and the drop-in import of ``from nn_conv import NNConv, NNConv_old``."""
import os
import pickle
import subprocess
import sys

import pytest
import torch

from oracle import golden
from tests import diag_oracle as D

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G8 = os.path.join(ROOT, 'tests', 'golden', 'g8_diag_nnconv.npz')


def _g8():
    return golden.load(G8)


def _cases(rec):
    for i in range(int(rec['n_cases'])):
        aggr, rw, bs, c = [str(v) for v in rec['c%d_case' % i]]
        yield i, aggr, rw == 'True', bs == 'True', int(c)


def _module(i, aggr, rw, bs, c, width=64, kin=3):
    from graph_pde_b200.nn_conv import DiagNNConv
    torch.manual_seed(100 + i)
    mlp = torch.nn.Sequential(torch.nn.Linear(kin, width), torch.nn.ReLU(), torch.nn.Linear(width, c))
    return DiagNNConv(c, c, mlp, aggr=aggr, root_weight=rw, bias=bs)


def test_oracle_matches_reference_outputs():
    rec = _g8()
    ei = torch.from_numpy(rec['edge_index'])
    ea = torch.from_numpy(rec['edge_attr']).double()
    for i, aggr, rw, bs, c in _cases(rec):
        p = 'c%d_' % i
        ws = [torch.from_numpy(rec[p + 'sd_nn.%d.weight' % l]).double() for l in (0, 2)]
        bb = [torch.from_numpy(rec[p + 'sd_nn.%d.bias' % l]).double() for l in (0, 2)]
        root = torch.from_numpy(rec[p + 'sd_root']).double() if rw else None
        bias = torch.from_numpy(rec[p + 'sd_bias']).double() if bs else None
        x = torch.from_numpy(rec['x'] if c > 1 else rec['x1']).double()
        out, _ = D.nnconv_diag_forward(x, ei, ea, ws, bb, root, bias, aggr)
        ref = torch.from_numpy(rec[p + 'out']).double()
        assert out.shape == ref.shape
        assert torch.allclose(out, ref, rtol=1e-5, atol=1e-6), (i, aggr, (out - ref).abs().max())


def test_init_stream_state_dict_and_repr_match_reference():
    rec = _g8()
    for i, aggr, rw, bs, c in _cases(rec):
        p = 'c%d_' % i
        conv = _module(i, aggr, rw, bs, c)
        sd = conv.state_dict()
        assert list(sd.keys()) == [str(k) for k in rec[p + 'keys']]
        for k, v in sd.items():
            assert torch.equal(v, torch.from_numpy(rec[p + 'sd_' + k])), (i, k)
        assert repr(conv).replace('DiagNNConv', 'NNConv') == str(rec[p + 'repr'])


@pytest.mark.parametrize('k,cin,cout', [(8, 4, 4), (4, 4, 8), (4, 8, 4), (16, 4, 4)])
def test_other_shapes_raise_before_any_launch(k, cin, cout):
    from graph_pde_b200.nn_conv import DiagNNConv
    mlp = torch.nn.Sequential(torch.nn.Linear(3, 8), torch.nn.ReLU(), torch.nn.Linear(8, k))
    conv = DiagNNConv(cin, cout, mlp)
    ei = torch.zeros(2, 5, dtype=torch.long)
    with pytest.raises(NotImplementedError) as err:
        conv(torch.zeros(3, cin), ei, torch.zeros(5, 3))
    assert all(str(v) in str(err.value) for v in (k, cin, cout))


def test_dropin_imports_both_names():
    code = ('from nn_conv import NNConv, NNConv_old, ECConv\n'
            'import torch, pickle\n'
            'mlp = torch.nn.Sequential(torch.nn.Linear(3, 8), torch.nn.ReLU(), torch.nn.Linear(8, 4))\n'
            'c = NNConv(4, 4, mlp, aggr="mean")\n'
            'assert type(c).__module__ == "nn_conv" and type(c).__qualname__ == "NNConv", type(c)\n'
            'assert repr(c) == "NNConv(4, 4)", repr(c)\n'
            'assert NNConv_old.__module__ == "nn_conv"\n'
            'import graph_pde_b200, torch_geometric.nn as tgnn\n'
            'assert ECConv is graph_pde_b200.NNConv and tgnn.NNConv is graph_pde_b200.NNConv\n'
            'assert graph_pde_b200.nn_conv.ECConv is graph_pde_b200.NNConv\n'
            'c2 = pickle.loads(pickle.dumps(c))\n'
            'assert type(c2) is NNConv\n'
            'print("ok")\n')
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, 'dropin'), ROOT]))
    res = subprocess.run([sys.executable, '-c', code], cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True)
    assert res.returncode == 0 and res.stdout.strip().endswith('ok'), res.stdout


def test_oracle_max_routes_gradient_to_winner():
    g = torch.Generator().manual_seed(3)
    ei = torch.tensor([[0, 1, 2, 0], [3, 3, 3, 1]])
    x = torch.randn(4, 2, dtype=torch.float64, generator=g, requires_grad=True)
    ea = torch.randn(4, 2, dtype=torch.float64, generator=g)
    ws = [torch.randn(5, 2, dtype=torch.float64, generator=g), torch.randn(2, 5, dtype=torch.float64, generator=g)]
    bs = [torch.randn(5, dtype=torch.float64, generator=g), torch.randn(2, dtype=torch.float64, generator=g)]
    out, am = D.nnconv_diag_forward(x, ei, ea, ws, bs, aggr='max')
    msg = D.messages(x, ei[0], ea, ws, bs)
    for o in range(2):
        w = am[3, o].item()
        assert msg[w, o] == msg[:3, o].max()
    assert (am[0] == -1).all() and (am[2] == -1).all()
    out[3].sum().backward()
    assert x.grad[3].abs().sum() == 0       # node 3 has no out-edges
