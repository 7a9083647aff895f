"""The Gaussian-kernel NNConv on the CPU: the fp64 oracle against the reference's own outputs and gradients (g11), the
module's init stream, state-dict keys and repr, every refusal, the drop-in import and pickle of
``nn_conv.NNConv_Gaussian``, and the bit budget of the exact probes of tests/gauss_probe.py."""
import os
import subprocess
import sys

import pytest
import torch

from oracle import golden
from tests import gauss_oracle as G
from tests import gauss_probe as GP

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G11 = os.path.join(ROOT, 'tests', 'golden', 'g11_gaussian_nnconv.npz')
C = 64


def _g11():
    return golden.load(G11)


def _cases(rec):
    for i in range(int(rec['n_cases'])):
        aggr, rw, bs, net = [str(v) for v in rec['c%d_case' % i]]
        yield i, aggr, rw == 'True', bs == 'True', net


def _nn(net):
    if net == 'linear':
        return torch.nn.Linear(1, C)
    return torch.nn.Sequential(torch.nn.Linear(1, 16), torch.nn.ReLU(), torch.nn.Linear(16, C))


def _module(i, aggr, rw, bs, net):
    from graph_pde_b200 import GaussianNNConv
    torch.manual_seed(200 + i)
    mlp = _nn(net)
    return GaussianNNConv(C, C, mlp, aggr=aggr, root_weight=rw, bias=bs)


def test_oracle_matches_reference_outputs_and_gradients():
    rec = _g11()
    ei = torch.from_numpy(rec['edge_index'])
    gw = torch.from_numpy(rec['gw']).double()
    for i, aggr, rw, bs, net in _cases(rec):
        p = 'c%d_' % i
        mlp = _nn(net).double()
        mlp.load_state_dict({k[len('nn.'):]: torch.from_numpy(rec[p + 'sd_' + k]).double()
                             for k in [str(k) for k in rec[p + 'keys']] if k.startswith('nn.')})
        root = torch.from_numpy(rec[p + 'sd_root']).double().requires_grad_() if rw else None
        bias = torch.from_numpy(rec[p + 'sd_bias']).double().requires_grad_() if bs else None
        x = torch.from_numpy(rec['x']).double().requires_grad_()
        ea = torch.from_numpy(rec['edge_attr']).double().requires_grad_()
        sigma = mlp(torch.ones(1, dtype=torch.float64))
        out, _ = G.gauss_forward(x, ei, ea, sigma, root, bias, aggr)
        ref = torch.from_numpy(rec[p + 'out']).double()
        assert out.shape == ref.shape
        assert torch.allclose(out, ref, rtol=1e-5, atol=1e-5), (i, aggr, (out - ref).abs().max())
        (out * gw).sum().backward()
        grads = {'x': x.grad, 'edge_attr': ea.grad}
        grads.update({'nn.' + k: v.grad for k, v in mlp.named_parameters()})
        if rw:
            grads['root'] = root.grad
        if bs:
            grads['bias'] = bias.grad
        for k, v in grads.items():
            r = torch.from_numpy(rec[p + 'grad_' + k]).double()
            scale = r.abs().max().clamp(min=1.0)
            assert (v - r).abs().max() / scale < 1e-5, (i, aggr, k, (v - r).abs().max())
        assert set('grad_' + k for k in grads) == {k[len(p):] for k in rec if k.startswith(p + 'grad_')}


def test_init_stream_state_dict_and_repr_match_reference():
    rec = _g11()
    for i, aggr, rw, bs, net in _cases(rec):
        p = 'c%d_' % i
        conv = _module(i, aggr, rw, bs, net)
        sd = conv.state_dict()
        assert list(sd.keys()) == [str(k) for k in rec[p + 'keys']]
        for k, v in sd.items():
            assert torch.equal(v, torch.from_numpy(rec[p + 'sd_' + k])), (i, k)
        assert repr(conv).replace('GaussianNNConv', 'NNConv_Gaussian') == str(rec[p + 'repr']) == 'NNConv_Gaussian(64, 64)'


@pytest.mark.parametrize('k,cin,cout', [(8, 4, 4), (4, 4, 8), (4, 8, 4), (16, 4, 4), (4097, 4097, 4097)])
def test_other_shapes_raise_before_any_launch(k, cin, cout):
    from graph_pde_b200 import GaussianNNConv
    conv = GaussianNNConv(cin, cout, torch.nn.Linear(1, k))
    with pytest.raises(NotImplementedError) as err:
        conv(torch.zeros(3, cin), torch.zeros(2, 5, dtype=torch.long), torch.ones(5, 3))
    assert all(str(v) in str(err.value) for v in (k, cin, cout))


@pytest.mark.parametrize('k_in', [1, 2])
def test_too_few_edge_attr_columns_raise(k_in):
    from graph_pde_b200 import GaussianNNConv
    conv = GaussianNNConv(4, 4, torch.nn.Linear(1, 4))
    ea = torch.ones(5) if k_in == 1 else torch.ones(5, k_in)
    with pytest.raises(ValueError, match='at least 3 columns'):
        conv(torch.zeros(3, 4), torch.zeros(2, 5, dtype=torch.long), ea)


def test_constructor_refusals():
    from graph_pde_b200 import GaussianNNConv
    lin = torch.nn.Linear(1, 4)
    with pytest.raises(ValueError, match='aggr'):
        GaussianNNConv(4, 4, lin, aggr='min')
    with pytest.raises(ValueError, match='flow'):
        GaussianNNConv(4, 4, lin, flow='sideways')
    with pytest.raises(ValueError, match='precision'):
        GaussianNNConv(4, 4, lin, precision='fp8')
    with pytest.raises(TypeError, match='unexpected keyword'):
        GaussianNNConv(4, 4, lin, normalize=True)
    for prec in ('f16', 'bf16', 'f16x2', 'fp32'):
        assert GaussianNNConv(4, 4, lin, precision=prec).precision == prec


def test_cpu_tensors_raise():
    from graph_pde_b200 import GaussianNNConv
    conv = GaussianNNConv(4, 4, torch.nn.Linear(1, 4))
    with pytest.raises(RuntimeError, match='must be a CUDA tensor'):
        conv(torch.zeros(3, 4), torch.zeros(2, 5, dtype=torch.long), torch.ones(5, 3))


def test_dropin_imports_all_three_names():
    code = ('from nn_conv import NNConv, NNConv_Gaussian, NNConv_old\n'
            'import torch, pickle\n'
            'import graph_pde_b200\n'
            'c = NNConv_Gaussian(64, 64, torch.nn.Linear(1, 64), aggr="mean")\n'
            'assert type(c).__module__ == "nn_conv" and type(c).__qualname__ == "NNConv_Gaussian", type(c)\n'
            'assert isinstance(c, graph_pde_b200.GaussianNNConv)\n'
            'assert repr(c) == "NNConv_Gaussian(64, 64)", repr(c)\n'
            'assert list(c.state_dict()) == ["root", "bias", "nn.weight", "nn.bias"], list(c.state_dict())\n'
            'c2 = pickle.loads(pickle.dumps(c))\n'
            'assert type(c2) is NNConv_Gaussian\n'
            'assert all(torch.equal(a, b) for a, b in zip(c.state_dict().values(), c2.state_dict().values()))\n'
            'assert NNConv.__module__ == "nn_conv" and NNConv_old.__module__ == "nn_conv"\n'
            'print("ok")\n')
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, 'dropin'), ROOT]))
    res = subprocess.run([sys.executable, '-c', code], cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True)
    assert res.returncode == 0 and res.stdout.strip().endswith('ok'), res.stdout


@pytest.mark.parametrize('aggr', ['add', 'max'])
@pytest.mark.parametrize('k_in', [3, 6])
def test_exact_probe_values_are_representable(aggr, k_in):
    """The probe's forward and every gradient evaluated in fp32 equal the fp64 evaluation exactly, and the values the
    kernels form stay on the grid the module docstring of tests/gauss_probe.py names."""
    ei = GP.graph(seed=1)
    ea = GP.edge_attr(ei.size(1), k_in, seed=1)
    lin = GP.nn_module(C, seed=1)
    x, gout, root, bias = GP.tensors(300, C, seed=1)
    a = 1 / torch.sqrt(torch.abs(ea[:, 1] * ea[:, 2]))
    assert torch.equal(torch.log2(a), torch.log2(a).round()) and a.min() >= 0.25 and a.max() <= 4
    sigma = lin(torch.ones(1)).detach().double()
    assert (sigma != 0).all() and torch.equal(sigma, sigma.round()) and sigma.abs().max() <= 4
    out64, am64, g64 = GP.reference(x, ei, ea, lin, root, bias, gout, aggr, torch.float64)
    out32, am32, g32 = GP.reference(x, ei, ea, lin, root, bias, gout, aggr, torch.float32)
    assert out64.abs().max() < 2 ** 22
    assert torch.equal(out32.double(), out64)
    if aggr == 'max':
        assert torch.equal(am32, am64)
    for k in g64:
        assert torch.equal(g32[k].double(), g64[k]), k
        assert g64[k].abs().max() < 2 ** 22, k
