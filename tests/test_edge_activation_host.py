"""Edge networks with LeakyReLU, ELU, Tanh or Sigmoid between their layers, on the CPU: the fp64 oracle against the
reference's own outputs (g10), how the library reads an edge network and which ones it refuses (and why), the drop-in
with a DenseNet of another activation, pickling and state-dict keys, and the bit budget of the exact LeakyReLU probe."""
import copy
import os
import pickle
import subprocess
import sys

import pytest
import torch

from oracle import golden
from tests import act_oracle as A
from tests import act_probe as AP

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G10 = os.path.join(ROOT, 'tests', 'golden', 'g10_edge_activations.npz')
MODULE_OF = {'leaky_relu': torch.nn.LeakyReLU, 'elu': torch.nn.ELU, 'tanh': torch.nn.Tanh, 'sigmoid': torch.nn.Sigmoid}


def _cases(rec):
    for i in range(int(rec['n_cases'])):
        kind, p, aggr = [str(v) for v in rec['c%d_case' % i]]
        yield i, kind, float(p), aggr


def _dense(dims, kind, p):
    from graph_pde_b200.models import DenseNet
    return DenseNet(dims, lambda: A.MODULES[kind](p))


def test_oracle_matches_reference_outputs():
    rec = golden.load(G10)
    ei = torch.from_numpy(rec['edge_index'])
    ea = torch.from_numpy(rec['edge_attr']).double()
    x = torch.from_numpy(rec['x']).double()
    for i, kind, p, aggr in _cases(rec):
        pre = 'c%d_' % i
        ws = [torch.from_numpy(rec[pre + 'sd_nn.layers.%d.weight' % l]).double() for l in (0, 2, 4)]
        bs = [torch.from_numpy(rec[pre + 'sd_nn.layers.%d.bias' % l]).double() for l in (0, 2, 4)]
        root = torch.from_numpy(rec[pre + 'sd_root']).double()
        bias = torch.from_numpy(rec[pre + 'sd_bias']).double()
        out, _ = A.nnconv_forward(x, ei, ea, ws, bs, root, bias, aggr, kind, p)
        ref = torch.from_numpy(rec[pre + 'out']).double()
        assert torch.allclose(out, ref, rtol=1e-5, atol=1e-6), (i, kind, aggr, float((out - ref).abs().max()))


def test_init_stream_and_state_dict_match_reference():
    """NNConv_old over models.DenseNet with the activation draws the reference's parameters and keys."""
    from graph_pde_b200.nn_conv import NNConv_old
    rec = golden.load(G10)
    for i, kind, p, aggr in _cases(rec):
        pre = 'c%d_' % i
        torch.manual_seed(1000 + i)
        conv = NNConv_old(8, 8, _dense([3, 16, 24, 64], kind, p), aggr=aggr)
        sd = conv.state_dict()
        assert list(sd.keys()) == [str(k) for k in rec[pre + 'keys']]
        for k, v in sd.items():
            assert torch.equal(v, torch.from_numpy(rec[pre + 'sd_' + k])), (i, k)


@pytest.mark.parametrize('module,spec', [
    (torch.nn.ReLU(), ('relu', 0.0)), (torch.nn.ReLU(inplace=True), ('relu', 0.0)),
    (torch.nn.LeakyReLU(), ('leaky_relu', 0.01)), (torch.nn.LeakyReLU(0.25, inplace=True), ('leaky_relu', 0.25)),
    (torch.nn.LeakyReLU(0.0), ('leaky_relu', 0.0)),
    (torch.nn.ELU(), ('elu', 1.0)), (torch.nn.ELU(alpha=0.5, inplace=True), ('elu', 0.5)),
    (torch.nn.Tanh(), ('tanh', 0.0)), (torch.nn.Sigmoid(), ('sigmoid', 0.0))])
def test_chain_recognition(module, spec):
    from graph_pde_b200.nn_conv import _edge_network
    mlp = torch.nn.Sequential(torch.nn.Linear(6, 16), module, torch.nn.Linear(16, 16), copy.deepcopy(module),
                              torch.nn.Linear(16, 64))
    lin, act = _edge_network(mlp)
    assert act == spec
    assert [l.out_features for l in lin] == [16, 16, 64]
    lin, act = _edge_network(torch.nn.Linear(6, 64))              # a single Linear uses no activation
    assert len(lin) == 1 and act == ('relu', 0.0)


def test_dense_net_with_each_activation():
    from graph_pde_b200.nn_conv import _edge_network
    for kind, p in [('leaky_relu', 0.2), ('elu', 0.7), ('tanh', 0.0), ('sigmoid', 0.0)]:
        lin, act = _edge_network(_dense([6, 32, 32, 64], kind, p))
        assert act == (kind, p) and len(lin) == 3


class DenseNet_sin(torch.nn.Module):
    """The multipole utilities' second network: Linear layers only, torch.sin applied inside forward()."""

    def __init__(self, layers):
        super().__init__()
        self.layers = torch.nn.ModuleList([torch.nn.Linear(a, b) for a, b in zip(layers[:-1], layers[1:])])

    def forward(self, x):
        for j, l in enumerate(self.layers):
            x = l(x)
            if j != len(self.layers) - 1:
                x = torch.sin(x)
        return x


def _seq(*mods):
    return torch.nn.Sequential(*mods)


L = torch.nn.Linear


@pytest.mark.parametrize('mlp,match', [
    (lambda: _seq(L(6, 16), torch.nn.Tanh(), L(16, 16), torch.nn.ReLU(), L(16, 64)), 'mixed activations'),
    (lambda: _seq(L(6, 16), torch.nn.LeakyReLU(0.1), L(16, 16), torch.nn.LeakyReLU(0.2), L(16, 64)),
     'mixed activations'),
    (lambda: _seq(L(6, 16), torch.nn.Tanh(), L(16, 64), torch.nn.Tanh()), 'no output nonlinearity'),
    (lambda: _seq(L(6, 16), torch.nn.BatchNorm1d(16), torch.nn.ReLU(), L(16, 64)), 'normalize=True'),
    (lambda: _seq(L(6, 16), torch.nn.GELU(), L(16, 64)), 'GELU is not supported: its derivative'),
    (lambda: _seq(L(6, 16), torch.nn.SiLU(), L(16, 64)), 'SiLU is not supported: its derivative'),
    (lambda: _seq(L(6, 16), torch.nn.Softplus(), L(16, 64)), 'Softplus is not supported: its derivative'),
    (lambda: DenseNet_sin([6, 16, 64]), 'DenseNet_sin'),
    (lambda: _seq(L(6, 16), L(16, 64)), 'two Linear layers without an activation'),
    (lambda: _seq(L(6, 16), torch.nn.LeakyReLU(-0.1), L(16, 64)), 'negative slope'),
    (lambda: _seq(L(6, 16), torch.nn.ELU(alpha=-1.0), L(16, 64)), 'negative alpha'),
    (lambda: _seq(L(6, 16), torch.nn.Tanh(), torch.nn.Tanh(), L(16, 64)), 'two activations in a row'),
    (lambda: _seq(torch.nn.Tanh(), L(6, 64)), 'must follow a Linear layer'),
    (lambda: _seq(L(6, 16), torch.nn.Dropout(), L(16, 64)), 'found Dropout')])
def test_refusals_name_the_reason(mlp, match):
    from graph_pde_b200.nn_conv import NNConv_old, _edge_network
    with pytest.raises(NotImplementedError, match=match):
        _edge_network(mlp())
    conv = NNConv_old(8, 8, mlp())
    with pytest.raises(NotImplementedError, match=match):
        conv._get_prepared('f16')                  # the first thing a forward does with the edge network


def test_out_nonlinearity_and_normalize_of_dense_net_are_refused():
    from graph_pde_b200.models import DenseNet
    from graph_pde_b200.nn_conv import _edge_network
    with pytest.raises(NotImplementedError, match='out_nonlinearity'):
        _edge_network(DenseNet([6, 16, 64], torch.nn.Tanh, out_nonlinearity=torch.nn.Tanh))
    bn = _seq(L(6, 16), torch.nn.BatchNorm1d(16), torch.nn.Tanh(), L(16, 64))
    with pytest.raises(NotImplementedError, match='normalize=True'):
        _edge_network(bn)


def test_prepared_weights_key_includes_the_activation(monkeypatch):
    """Swapping the activation module of a conv (same parameters) prepares new weights."""
    from graph_pde_b200 import nn_conv
    made = []

    class FakePrepared(object):
        def __init__(self, linears, cin, cout, precision, act):
            made.append(act)
    monkeypatch.setattr(nn_conv, '_Prepared', FakePrepared)
    conv = nn_conv.NNConv_old(8, 8, _dense([6, 16, 64], 'tanh', 0.0))
    conv._get_prepared('f16')
    conv._get_prepared('f16')
    conv.nn.layers[1] = torch.nn.Sigmoid()
    conv._get_prepared('f16')
    assert made == [('tanh', 0.0), ('sigmoid', 0.0)]


def test_dropin_with_a_dense_net_of_another_activation():
    """``from nn_conv import NNConv_old`` with a DenseNet(..., torch.nn.Tanh) edge network, as a reference script
    writes it: the module accepts it and keeps the reference's state-dict keys."""
    code = ('import torch; from nn_conv import NNConv_old; from graph_pde_b200.models import DenseNet; '
            'from graph_pde_b200.nn_conv import _edge_network; '
            'conv = NNConv_old(16, 16, DenseNet([6, 64, 64, 256], torch.nn.Tanh), aggr="mean"); '
            'assert _edge_network(conv.nn)[1] == ("tanh", 0.0); '
            'print("keys", ",".join(conv.state_dict().keys()))')
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, 'dropin'), ROOT]))
    res = subprocess.run([sys.executable, '-c', code], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True, cwd=ROOT)
    assert res.returncode == 0, res.stdout
    assert 'keys root,bias,nn.layers.0.weight,nn.layers.0.bias,nn.layers.2.weight,nn.layers.2.bias,' \
           'nn.layers.4.weight,nn.layers.4.bias' in res.stdout


@pytest.mark.parametrize('kind,p', [('leaky_relu', 0.3), ('elu', 0.5), ('tanh', 0.0), ('sigmoid', 0.0)])
def test_pickle_roundtrip_keeps_the_activation(kind, p, tmp_path):
    from graph_pde_b200.nn_conv import DiagNNConv, NNConv_old, _edge_network
    for conv in (NNConv_old(8, 8, _dense([6, 16, 64], kind, p)), DiagNNConv(8, 8, _dense([6, 16, 8], kind, p))):
        path = tmp_path / 'm.pt'
        torch.save(conv, path)
        back = torch.load(path, weights_only=False)
        assert _edge_network(back.nn)[1] == (kind, p)
        assert isinstance(back.nn.layers[1], MODULE_OF[kind])
        assert list(back.state_dict().keys()) == list(conv.state_dict().keys())
        for a, b in zip(conv.state_dict().values(), back.state_dict().values()):
            assert torch.equal(a, b)
        assert pickle.loads(pickle.dumps(conv.nn.layers[1])).__class__ is MODULE_OF[kind]


def test_derivatives_from_the_output_match_autograd():
    """GRADS[kind](f(z)) is torch's derivative, including at z = 0 (LeakyReLU: the slope, ELU: alpha)."""
    z = torch.cat([torch.linspace(-6, 6, 1001, dtype=torch.float64), torch.zeros(1, dtype=torch.float64)])
    for kind, p in [('relu', 0.0), ('leaky_relu', 0.25), ('elu', 0.7), ('tanh', 0.0), ('sigmoid', 0.0)]:
        zz = z.clone().requires_grad_()
        y = A.MODULES[kind](p).double()(zz)
        y.sum().backward()
        assert torch.allclose(A.GRADS[kind](y.detach(), p), zz.grad, rtol=1e-12, atol=1e-12), kind
        assert torch.allclose(A.ACTS[kind](z, p), y.detach(), rtol=1e-12, atol=1e-15), kind


@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2', 'fp32'])
def test_exact_probe_budget(precision):
    """The LeakyReLU(0.25) probe of test_gpu_edge_activation.py is exact at ``precision``, and its pre-activations take
    both signs (and zero) in both hidden layers."""
    ei, n = AP.graph()
    pr = AP.make(ei, n, precision=precision)
    zs = AP.assert_exact(pr, precision)
    for z in zs:
        assert int((z < 0).sum()) > 100 and int((z > 0).sum()) > 100 and int((z == 0).sum()) > 0


def test_probe_budget_is_tight_enough_to_fail():
    """The proof rejects the same probe with every output-gradient row at bf16 (the hub's dY needs more than 8 bits)."""
    ei, n = AP.graph()
    from tests import probes as P
    pr = P.make_probe(ei, n, AP.LAYERS, 64, 64, seed=3, T=2, grad=True)
    with pytest.raises(P.NotExact, match='dY'):
        AP.assert_exact(pr, 'bf16')
