"""Edge networks with Hardtanh, ReLU6, Hardsigmoid, SELU, CELU, Softsign or LogSigmoid between their layers, on the CPU:
the fp64 oracle against the reference's own outputs and gradients (g14), how the library reads each module, the
refusals, the C-side parameter validation (no device needed), and the drop-in, pickling and state-dict keys."""
import copy
import ctypes
import os
import pickle
import subprocess
import sys

import pytest
import torch

from oracle import golden
from tests import act_more_oracle as AM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G14 = os.path.join(ROOT, 'tests', 'golden', 'g14_edge_activations_more.npz')
L = torch.nn.Linear
KINDS = [('relu6', None), ('hardtanh', (-0.3, 0.7)), ('hardsigmoid', None), ('selu', None), ('celu', 0.5),
         ('softsign', None), ('logsigmoid', None)]


def _param(kind, s):
    if s == 'None':
        return None
    if kind == 'hardtanh':
        return tuple(float(v) for v in s.split(','))
    return float(s)


def _cases(rec):
    for i in range(int(rec['n_cases'])):
        kind, p, aggr = [str(v) for v in rec['c%d_case' % i]]
        yield i, kind, _param(kind, p), aggr


def _dense(dims, kind, p):
    from graph_pde_b200.models import DenseNet
    return DenseNet(dims, lambda: AM.MODULES[kind](p))


def test_oracle_matches_reference_outputs_and_gradients():
    rec = golden.load(G14)
    ei = torch.from_numpy(rec['edge_index'])
    g = torch.from_numpy(rec['grad_out']).double()
    seen = set()
    for i, kind, p, aggr in _cases(rec):
        seen.add(kind)
        pre = 'c%d_' % i
        ws = [torch.from_numpy(rec[pre + 'sd_nn.layers.%d.weight' % l]).double().requires_grad_() for l in (0, 2, 4)]
        bs = [torch.from_numpy(rec[pre + 'sd_nn.layers.%d.bias' % l]).double().requires_grad_() for l in (0, 2, 4)]
        root = torch.from_numpy(rec[pre + 'sd_root']).double().requires_grad_()
        bias = torch.from_numpy(rec[pre + 'sd_bias']).double().requires_grad_()
        ea = torch.from_numpy(rec['edge_attr']).double().requires_grad_()
        x = torch.from_numpy(rec['x']).double().requires_grad_()
        out, _ = AM.nnconv_forward(x, ei, ea, ws, bs, root, bias, aggr, kind, p)
        ref = torch.from_numpy(rec[pre + 'out']).double()
        assert torch.allclose(out, ref, rtol=1e-5, atol=1e-5), (i, kind, aggr, float((out - ref).abs().max()))
        (out * g).sum().backward()
        got = {'x': x.grad, 'edge_attr': ea.grad, 'root': root.grad, 'bias': bias.grad}
        for j, l in enumerate((0, 2, 4)):
            got['nn.layers.%d.weight' % l] = ws[j].grad
            got['nn.layers.%d.bias' % l] = bs[j].grad
        for k, v in got.items():
            r = torch.from_numpy(rec[pre + 'grad_' + k]).double()
            assert torch.allclose(v, r, rtol=1e-4, atol=1e-5), (i, kind, aggr, k, float((v - r).abs().max()))
    assert seen == {k for k, _ in KINDS}


def test_fixture_saturates_the_clamps():
    """Both bounds of every clamp are reached on some edges of g14's first hidden layer, so its gradients test the
    kinks."""
    rec = golden.load(G14)
    ea = torch.from_numpy(rec['edge_attr']).double()
    for i, kind, p, aggr in _cases(rec):
        if kind not in ('relu6', 'hardtanh', 'hardsigmoid'):
            continue
        pre = 'c%d_' % i
        w = torch.from_numpy(rec[pre + 'sd_nn.layers.0.weight']).double()
        b = torch.from_numpy(rec[pre + 'sd_nn.layers.0.bias']).double()
        y = AM.MODULES[kind](p)(torch.nn.functional.linear(ea, w, b))
        lo, hi = {'relu6': (0, 6), 'hardtanh': p, 'hardsigmoid': (0, 1)}[kind]
        assert int((y == lo).sum()) > 0 and int((y > lo).sum()) > 0, (kind, 'lo')
        if kind != 'relu6':
            assert int((y == hi).sum()) > 0, (kind, 'hi')


def test_reference_state_dict_keys():
    from graph_pde_b200.nn_conv import NNConv_old
    rec = golden.load(G14)
    for i, kind, p, aggr in _cases(rec):
        conv = NNConv_old(8, 8, _dense([3, 16, 24, 64], kind, p), aggr=aggr)
        assert list(conv.state_dict().keys()) == [str(k) for k in rec['c%d_keys' % i]]


@pytest.mark.parametrize('module,spec', [
    (torch.nn.ReLU6(), ('clamp', (1.0, 0.0, 0.0, 6.0))), (torch.nn.ReLU6(inplace=True), ('clamp', (1.0, 0.0, 0.0, 6.0))),
    (torch.nn.Hardtanh(), ('clamp', (1.0, 0.0, -1.0, 1.0))),
    (torch.nn.Hardtanh(-0.3, 0.7, inplace=True), ('clamp', (1.0, 0.0, -0.3, 0.7))),
    (torch.nn.Hardtanh(0.0, 6.0), ('clamp', (1.0, 0.0, 0.0, 6.0))),
    (torch.nn.Hardsigmoid(), ('clamp', (1.0 / 6.0, 0.5, 0.0, 1.0))),
    (torch.nn.Hardsigmoid(inplace=True), ('clamp', (1.0 / 6.0, 0.5, 0.0, 1.0))),
    (torch.nn.SELU(), ('scaled_elu', (1.0507009873554805, 1.6732632423543772, 1.0))),
    (torch.nn.SELU(inplace=True), ('scaled_elu', (1.0507009873554805, 1.6732632423543772, 1.0))),
    (torch.nn.CELU(), ('scaled_elu', (1.0, 1.0, 1.0))), (torch.nn.CELU(0.5, inplace=True), ('scaled_elu', (1.0, 0.5, 2.0))),
    (torch.nn.Softsign(), ('softsign', ())), (torch.nn.LogSigmoid(), ('logsigmoid', ()))])
def test_chain_recognition(module, spec):
    from graph_pde_b200.nn_conv import _edge_network
    mlp = torch.nn.Sequential(L(6, 16), module, L(16, 16), copy.deepcopy(module), L(16, 64))
    lin, act = _edge_network(mlp)
    assert act == spec
    assert [l.out_features for l in lin] == [16, 16, 64]


@pytest.mark.parametrize('kind,p', KINDS)
def test_dense_net_with_each_activation(kind, p):
    from graph_pde_b200.nn_conv import _edge_network
    lin, act = _edge_network(_dense([6, 32, 32, 64], kind, p))
    assert act == AM.SPECS[kind](p) and len(lin) == 3


def test_relu6_and_hardtanh_0_6_are_one_activation():
    """ReLU6 is torch's Hardtanh(0, 6): a network with both is one activation, not a mixed one."""
    from graph_pde_b200.nn_conv import _edge_network
    mlp = torch.nn.Sequential(L(6, 16), torch.nn.ReLU6(), L(16, 16), torch.nn.Hardtanh(0.0, 6.0), L(16, 64))
    assert _edge_network(mlp)[1] == ('clamp', (1.0, 0.0, 0.0, 6.0))


def _seq(*mods):
    return torch.nn.Sequential(*mods)


@pytest.mark.parametrize('mlp,match', [
    (lambda: _seq(L(6, 16), torch.nn.CELU(0.0), L(16, 64)), 'CELU with alpha <= 0'),
    (lambda: _seq(L(6, 16), torch.nn.CELU(-0.5), L(16, 64)), 'CELU with alpha <= 0'),
    (lambda: _seq(L(6, 16), torch.nn.Hardtanh(0.0, 6.0), L(16, 16), torch.nn.Hardtanh(0.0, 5.0), L(16, 64)),
     'mixed activations'),
    (lambda: _seq(L(6, 16), torch.nn.SELU(), L(16, 16), torch.nn.ELU(), L(16, 64)), 'mixed activations'),
    (lambda: _seq(L(6, 16), torch.nn.CELU(1.0), L(16, 16), torch.nn.ELU(1.0), L(16, 64)), 'mixed activations'),
    (lambda: _seq(L(6, 16), torch.nn.Softsign(), L(16, 64), torch.nn.Softsign()), 'no output nonlinearity'),
    (lambda: _seq(L(6, 16), torch.nn.Hardshrink(), L(16, 64)), r'LogSigmoid between them .* found Hardshrink$')])
def test_refusals_name_the_reason(mlp, match):
    from graph_pde_b200.nn_conv import NNConv_old, _edge_network
    with pytest.raises(NotImplementedError, match=match):
        _edge_network(mlp())
    conv = NNConv_old(8, 8, mlp())
    with pytest.raises(NotImplementedError, match=match):
        conv._get_prepared('f16')


def _lib_or_skip():
    from graph_pde_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip('libnnconv_b200.so is not built')
    return _lib, _lib.lib()


@pytest.mark.parametrize('kind,params', [
    ('clamp', (1.0, 0.0, 6.0, 6.0)), ('clamp', (1.0, 0.0, 1.0, 0.0)), ('clamp', (0.0, 0.0, 0.0, 6.0)),
    ('clamp', (-1.0, 0.0, 0.0, 6.0)), ('clamp', (1.0, 0.0, float('-inf'), 6.0)), ('clamp', (1.0, float('nan'), 0.0, 6.0)),
    ('clamp', (1.0, 0.0, 6.0)), ('scaled_elu', (0.0, 1.0, 1.0)), ('scaled_elu', (1.0, -0.1, 1.0)),
    ('scaled_elu', (1.0, 1.0, 0.0)), ('scaled_elu', (1.0, float('inf'), 1.0)), ('scaled_elu', (1.0, 1.0)),
    ('softsign', (1.0, 2.0)), ('clamp', ()), (99, ())])
def test_abi_refuses_bad_parameters_before_any_device_work(kind, params):
    """nnconv_weights_create_act_params and its diagonal twin refuse with NNCONV_ERR_ARG, naming the reason, before
    they touch the weights (null device pointers here) or the device."""
    _lib, Lb = _lib_or_skip()
    dims = (ctypes.c_int * 4)(6, 16, 16, 64)
    code = _lib.ACT[kind] if isinstance(kind, str) else kind
    q = (ctypes.c_float * max(len(params), 1))(*params)
    null = (ctypes.c_void_p * 3)()
    h = ctypes.c_void_p()
    st = Lb.nnconv_weights_create_act_params(3, dims, 8, 8, _lib.PREC['f16'], code, q, len(params), null, null, None,
                                             0, None, ctypes.byref(h))
    assert st == 1 and not h.value, st           # NNCONV_ERR_ARG
    assert b'activation' in Lb.nnconv_last_error()
    st = Lb.nnconv_diag_weights_create_act_params(3, dims, 64, _lib.PREC['f16'], code, q, len(params), null, null,
                                                  None, 0, None, ctypes.byref(h))
    assert st == 1 and not h.value, st


def test_abi_single_parameter_call_refuses_the_block_kinds():
    """nnconv_weights_create_act is the one-parameter case: a clamp or scaled ELU needs its whole block."""
    _lib, Lb = _lib_or_skip()
    dims = (ctypes.c_int * 4)(6, 16, 16, 64)
    null = (ctypes.c_void_p * 3)()
    h = ctypes.c_void_p()
    for kind in ('clamp', 'scaled_elu'):
        st = Lb.nnconv_weights_create_act(3, dims, 8, 8, 1, _lib.ACT[kind], 1.0, null, null, None, 0, None,
                                          ctypes.byref(h))
        assert st == 1 and b'takes' in Lb.nnconv_last_error(), kind


def test_abi_constants_match_the_header():
    from graph_pde_b200 import _lib
    with open(os.path.join(ROOT, 'include', 'nnconv_b200.h')) as f:
        hdr = f.read()
    for kind, code in _lib.ACT.items():
        assert '#define NNCONV_ACT_%s %d\n' % (kind.upper(), code) in hdr, kind


def test_derivatives_from_the_output_match_autograd():
    """GRADS[kind](f(z)) is torch's derivative in fp64, including at the bounds of the clamps and at z = 0."""
    z = torch.cat([torch.linspace(-8, 8, 1601, dtype=torch.float64),
                   torch.tensor([0.0, 6.0, -0.3, 0.7, 3.0, -3.0, -1.0, 1.0], dtype=torch.float64)])
    for kind, p in KINDS:
        zz = z.clone().requires_grad_()
        y = AM.MODULES[kind](p).double()(zz)
        y.sum().backward()
        assert torch.allclose(AM.GRADS[kind](y.detach(), p), zz.grad, rtol=1e-7, atol=1e-12), kind


def test_prepared_weights_key_includes_the_parameters(monkeypatch):
    """Hardtanh(0, 6) -> ReLU6 reuses the prepared weights (one spec); Hardtanh(0, 5) prepares new ones."""
    from graph_pde_b200 import nn_conv
    made = []

    class FakePrepared(object):
        def __init__(self, linears, cin, cout, precision, act):
            made.append(act)
    monkeypatch.setattr(nn_conv, '_Prepared', FakePrepared)
    conv = nn_conv.NNConv_old(8, 8, _dense([6, 16, 64], 'hardtanh', (0.0, 6.0)))
    conv._get_prepared('f16')
    conv.nn.layers[1] = torch.nn.ReLU6()
    conv._get_prepared('f16')
    conv.nn.layers[1] = torch.nn.Hardtanh(0.0, 5.0)
    conv._get_prepared('f16')
    assert made == [('clamp', (1.0, 0.0, 0.0, 6.0)), ('clamp', (1.0, 0.0, 0.0, 5.0))]


def test_dropin_with_a_dense_net_of_relu6_and_selu():
    """``from nn_conv import NNConv_old`` with DenseNet(..., torch.nn.ReLU6) and SELU edge networks, as a reference
    script writes them."""
    code = ('import torch; from nn_conv import NNConv_old; from graph_pde_b200.models import DenseNet; '
            'from graph_pde_b200.nn_conv import _edge_network; '
            'conv = NNConv_old(16, 16, DenseNet([6, 64, 64, 256], torch.nn.ReLU6), aggr="mean"); '
            'assert _edge_network(conv.nn)[1] == ("clamp", (1.0, 0.0, 0.0, 6.0)); '
            'conv2 = NNConv_old(16, 16, DenseNet([6, 64, 64, 256], torch.nn.SELU), aggr="mean"); '
            'assert _edge_network(conv2.nn)[1][0] == "scaled_elu"; '
            'print("keys", ",".join(conv.state_dict().keys()))')
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, 'dropin'), ROOT]))
    res = subprocess.run([sys.executable, '-c', code], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True, cwd=ROOT)
    assert res.returncode == 0, res.stdout
    assert 'keys root,bias,nn.layers.0.weight,nn.layers.0.bias,nn.layers.2.weight,nn.layers.2.bias,' \
           'nn.layers.4.weight,nn.layers.4.bias' in res.stdout


@pytest.mark.parametrize('kind,p', KINDS)
def test_pickle_roundtrip_keeps_the_activation(kind, p, tmp_path):
    from graph_pde_b200.nn_conv import DiagNNConv, NNConv_old, _edge_network
    for conv in (NNConv_old(8, 8, _dense([6, 16, 64], kind, p)), DiagNNConv(8, 8, _dense([6, 16, 8], kind, p))):
        path = tmp_path / 'm.pt'
        torch.save(conv, path)
        back = torch.load(path, weights_only=False)
        assert _edge_network(back.nn)[1] == AM.SPECS[kind](p)
        assert type(back.nn.layers[1]) is type(conv.nn.layers[1])
        assert list(back.state_dict().keys()) == list(conv.state_dict().keys())
        for a, b in zip(conv.state_dict().values(), back.state_dict().values()):
            assert torch.equal(a, b)
        assert pickle.loads(pickle.dumps(conv.nn.layers[1])).__class__ is type(conv.nn.layers[1])
