"""Edge networks whose hidden activation is ReLU6, Hardtanh(-0.3, 0.7), Hardsigmoid, SELU, CELU(0.5), Softsign or
LogSigmoid, on the GPU: the matrix of tests/test_gpu_edge_activation.py (forward parity on every application path and
precision, gradients against fp64 autograd on every backward path, the kernels that run, CUDA-graph replay, fp16 range
reporting), and the bound probe of the clamps: hidden units whose pre-activation is an exact fp32 number at, one ulp
inside, well inside and beyond a bound, whose gradients are zero exactly where fp64 torch's are, at every precision.
pytest -m gpu."""
import pytest
import torch

from tests import act_more_oracle as AM
from tests.helpers import TOL, rel_err
from tests.test_gpu_edge_activation import (C, DIMS, GTOL, _ea_index, _hub_graph, _inputs,
                                            _library_grads, _low_degree_graph, _template_args, formulation)  # noqa: F401

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ACTS = [('relu6', None), ('hardtanh', (-0.3, 0.7)), ('hardsigmoid', None), ('selu', None), ('celu', 0.5),
        ('softsign', None), ('logsigmoid', None)]
PRECS = ['f16', 'bf16', 'f16x2', 'fp32']
CODE = {'relu6': 5, 'hardtanh': 5, 'hardsigmoid': 5, 'selu': 6, 'celu': 6, 'softsign': 7, 'logsigmoid': 8}


def _mlp(dims, kind, p):
    from graph_pde_b200.models import DenseNet
    return DenseNet(dims, lambda: AM.MODULES[kind](p))


def _conv(kind, p, precision, aggr='add', seed=0, cls=None, dims=DIMS, **kw):
    """The conv with its first layer scaled by 4, so that the clamps saturate on a good share of the edges."""
    from graph_pde_b200.nn_conv import NNConv_old
    torch.manual_seed(seed)
    conv = (cls or NNConv_old)(C, C, _mlp(dims, kind, p), aggr=aggr, precision=precision, **kw)
    with torch.no_grad():
        conv.nn.layers[0].weight.mul_(4.0)
    return conv.to(DEV)


def _params(conv):
    lin = [m for m in conv.nn.layers if isinstance(m, torch.nn.Linear)]
    return ([l.weight.detach().double().cpu() for l in lin], [l.bias.detach().double().cpu() for l in lin],
            conv.root.detach().double().cpu(), conv.bias.detach().double().cpu())


def _oracle_out(conv, kind, p, x, ei, ea, aggr, diag=False):
    ws, bs, root, bias = _params(conv)
    if diag:
        return AM.diag_forward(x.double(), ei, ea.double(), ws, bs, root, bias, aggr, kind, p)
    return AM.nnconv_forward(x.double(), ei, ea.double(), ws, bs, root, bias, aggr, kind, p)[0]


def _reference_grads(conv, kind, p, ei, ea, xs, gs, diag=False, ws=None, bs=None):
    w0, b0, root, bias = _params(conv)
    ws, bs = ws or w0, bs or b0
    leaves = [w.requires_grad_() for w in ws] + [b.requires_grad_() for b in bs] + [root.requires_grad_(),
                                                                                   bias.requires_grad_()]
    ea64 = ea.double().requires_grad_()
    x64 = [x.double().requires_grad_() for x in xs]
    loss = 0
    for x, g in zip(x64, gs):
        if diag:
            out = AM.diag_forward(x, ei, ea64, ws, bs, root, bias, conv.aggr, kind, p)
        else:
            out = AM.nnconv_forward(x, ei, ea64, ws, bs, root, bias, conv.aggr, kind, p)[0]
        loss = loss + (out * g.double()).sum()
    loss.backward()
    return [l.grad for l in leaves] + [ea64.grad] + [x.grad for x in x64]


def _check_grads(conv, kind, p, ei, ea, xs, gs, precision, what, diag=False):
    got = _library_grads(conv, ei, ea, xs, gs)
    ref = _reference_grads(conv, kind, p, ei, ea, xs, gs, diag)
    k_ea = _ea_index(conv)
    for i, (a, b) in enumerate(zip(got, ref)):
        err = rel_err(a, b)
        tol = 0.3 if (i == k_ea and precision in ('f16', 'bf16')) else GTOL[precision]
        assert err < tol, (kind, what, i, err)
    return got


# ---- forward parity ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('aggr', ['add', 'mean', 'max'])
@pytest.mark.parametrize('precision', PRECS)
@pytest.mark.parametrize('kind,p', ACTS)
def test_forward_cached(kind, p, precision, aggr, formulation):
    formulation('off')
    ei, n = _hub_graph()
    ea, (x,), _ = _inputs(ei, n)
    conv = _conv(kind, p, precision, aggr)
    with torch.no_grad():
        out = conv(x.to(DEV), ei.to(DEV), ea.to(DEV))
    err = rel_err(out, _oracle_out(conv, kind, p, x, ei, ea, aggr))
    assert err < TOL[precision], (kind, precision, aggr, err)


@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2'])
@pytest.mark.parametrize('kind,p', ACTS)
def test_forward_streamed_prefix_inside_a_hub(kind, p, precision, formulation):
    from graph_pde_b200 import nn_conv
    formulation('off')
    ei, n = _hub_graph()
    ea, (x,), _ = _inputs(ei, n)
    conv = _conv(kind, p, precision, 'mean')
    with torch.no_grad():
        cached = conv(x.to(DEV), ei.to(DEV), ea.to(DEV))
    conv.edge_feature_bytes = 12032 * 128 * 2 * (2 if precision == 'f16x2' else 1) // 3
    conv.invalidate()
    s0 = nn_conv.stats['streamed_chunk_passes']
    with torch.no_grad():
        out = conv(x.to(DEV), ei.to(DEV), ea.to(DEV))
    assert nn_conv.stats['streamed_chunk_passes'] > s0
    assert 0 < next(iter(conv._h_cache.values())).E_res < 6000
    assert rel_err(out, cached) < 1e-5
    assert rel_err(out, _oracle_out(conv, kind, p, x, ei, ea, 'mean')) < TOL[precision]


@pytest.mark.parametrize('precision', ['f16', 'bf16'])
@pytest.mark.parametrize('kind,p', ACTS)
def test_forward_formulation_b(kind, p, precision, formulation):
    from graph_pde_b200 import nn_conv
    formulation('on')
    ei, n = _low_degree_graph()
    ea, (x,), _ = _inputs(ei, n)
    conv = _conv(kind, p, precision, 'mean')
    k0 = nn_conv.stats['edge_kernel_passes']
    with torch.no_grad():
        out = conv(x.to(DEV), ei.to(DEV), ea.to(DEV))
    assert nn_conv.stats['edge_kernel_passes'] > k0
    assert rel_err(out, _oracle_out(conv, kind, p, x, ei, ea, 'mean')) < TOL[precision]


@pytest.mark.parametrize('aggr', ['add', 'mean', 'max'])
@pytest.mark.parametrize('precision', PRECS)
@pytest.mark.parametrize('kind,p', ACTS)
def test_forward_diag(kind, p, precision, aggr):
    from graph_pde_b200.nn_conv import DiagNNConv
    ei, n = _hub_graph()
    ea, (x,), _ = _inputs(ei, n)
    conv = _conv(kind, p, precision, aggr, cls=DiagNNConv, dims=[6, 128, 128, C])
    with torch.no_grad():
        out = conv(x.to(DEV), ei.to(DEV), ea.to(DEV))
    err = rel_err(out, _oracle_out(conv, kind, p, x, ei, ea, aggr, diag=True))
    assert err < TOL[precision], (kind, precision, aggr, err)


@pytest.mark.parametrize('precision', PRECS)
@pytest.mark.parametrize('kind,p', ACTS)
def test_forward_bipartite(kind, p, precision, formulation):
    """Messages from 400 sources into 300 targets: the union-graph oracle's target rows."""
    formulation('off')
    ei, n = _hub_graph()
    ea, (x,), _ = _inputs(ei, n)
    n_dst = 300
    ei = torch.stack([ei[0], ei[1] % n_dst])
    x_dst = torch.randn(n_dst, C, generator=torch.Generator().manual_seed(5))
    conv = _conv(kind, p, precision, 'mean')
    with torch.no_grad():
        out = conv((x.to(DEV), x_dst.to(DEV)), ei.to(DEV), ea.to(DEV))
    xu = torch.cat([x, x_dst])
    eu = torch.stack([ei[0], ei[1] + n])
    ref = _oracle_out(conv, kind, p, xu, eu, ea, 'mean')[n:]
    assert out.shape == (n_dst, C)
    assert rel_err(out, ref) < TOL[precision], (kind, precision)


# ---- gradients ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('T', [1, 6])
@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2'])
@pytest.mark.parametrize('kind,p', ACTS)
def test_tensor_core_backward(kind, p, precision, T, formulation):
    """Kept activations and recomputed ones: both against fp64 autograd, and against each other."""
    from graph_pde_b200 import nn_conv
    formulation('off')
    ei, n = _hub_graph(e=6000, hub=2000)
    ea, xs, gs = _inputs(ei, n, T=T)
    conv = _conv(kind, p, precision, 'mean')
    b0 = nn_conv.stats['mlp_backwards']
    kept = _check_grads(conv, kind, p, ei, ea, xs, gs, precision, 'kept')
    assert nn_conv.stats['mlp_backwards'] > b0
    conv.zero_grad(set_to_none=True)
    conv.invalidate()
    old = nn_conv._KEEP_ACTS_MAX_BYTES
    nn_conv._KEEP_ACTS_MAX_BYTES = 0
    try:
        recomputed = _check_grads(conv, kind, p, ei, ea, xs, gs, precision, 'recomputed')
    finally:
        nn_conv._KEEP_ACTS_MAX_BYTES = old
    for a, b in zip(kept, recomputed):
        assert rel_err(a, b) < 1e-5


@pytest.mark.parametrize('precision', ['f16', 'f16x2'])
@pytest.mark.parametrize('kind,p', ACTS)
def test_streamed_training(kind, p, precision, formulation):
    from graph_pde_b200 import nn_conv
    formulation('off')
    ei, n = _hub_graph()
    ea, xs, gs = _inputs(ei, n, T=2)
    h_bytes = 12032 * 128 * 2 * (2 if precision == 'f16x2' else 1)
    conv = _conv(kind, p, precision, 'add', edge_feature_bytes=h_bytes // 3, streamed_training=True)
    s0 = nn_conv.stats['streamed_backward_chunk_passes']
    _check_grads(conv, kind, p, ei, ea, xs, gs, precision, 'streamed')
    assert nn_conv.stats['streamed_backward_chunk_passes'] > s0


@pytest.mark.parametrize('precision', ['fp32', 'f16'])
@pytest.mark.parametrize('kind,p', ACTS)
def test_cuda_core_backward(kind, p, precision, monkeypatch):
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_BWD_MODE', 'fp32')
    ei, n = _hub_graph(e=4000, hub=1000)
    ea, xs, gs = _inputs(ei, n, T=2)
    conv = _conv(kind, p, precision, 'mean')
    _check_grads(conv, kind, p, ei, ea, xs, gs, 'fp32', 'cuda cores')


@pytest.mark.parametrize('precision', ['f16', 'fp32'])
@pytest.mark.parametrize('kind,p', ACTS)
def test_diag_backward(kind, p, precision):
    from graph_pde_b200.nn_conv import DiagNNConv
    ei, n = _hub_graph(e=4000, hub=1000)
    ea, xs, gs = _inputs(ei, n, T=2)
    conv = _conv(kind, p, precision, 'add', cls=DiagNNConv, dims=[6, 128, 128, C])
    got = _library_grads(conv, ei, ea, xs, gs)
    ref = _reference_grads(conv, kind, p, ei, ea, xs, gs, diag=True)
    for i, (a, b) in enumerate(zip(got, ref)):
        assert rel_err(a, b) < (3e-2 if precision == 'f16' else 1e-4), (kind, i, rel_err(a, b))


# ---- the bound probe of the clamps -------------------------------------------------------------------------------------
def _bound_biases(lo, hi):
    """fp32 pre-activations at, one ulp inside, well inside and beyond each bound."""
    f = torch.float32
    lo_t, hi_t = torch.tensor(lo, dtype=f), torch.tensor(hi, dtype=f)
    inf = torch.tensor(float('inf'), dtype=f)
    vals = [lo_t, torch.nextafter(lo_t, inf), torch.nextafter(torch.nextafter(lo_t, inf), inf), hi_t,
            torch.nextafter(hi_t, -inf), torch.nextafter(torch.nextafter(hi_t, -inf), -inf), (lo_t + hi_t) / 2,
            lo_t - 1, hi_t + 1, lo_t + (hi_t - lo_t) / 64, hi_t - (hi_t - lo_t) / 64]
    return torch.stack(vals)


def _bound_probe_conv(kind, p, precision, **kw):
    """Hidden units 0..10 of the second hidden layer have a zero weight row and an fp32 bias from _bound_biases, so
    their pre-activation is that bias exactly on every edge at every precision (the GEMM epilogue adds the bias to a
    zero accumulator in fp32)."""
    conv = _conv(kind, p, precision, 'mean', dims=[6, 128, 128, C * C], **kw)
    lo, hi = (0.0, 6.0) if kind == 'relu6' else p
    b = _bound_biases(lo, hi)
    with torch.no_grad():
        conv.nn.layers[2].weight[:b.numel()] = 0
        conv.nn.layers[2].bias[:b.numel()] = b.to(DEV)
    return conv


def _check_bound_units(conv, kind, p, ei, ea, xs, gs, precision, what):
    """The probed units against fp64 autograd: their bias gradient is 0 exactly where torch's is (at and beyond a
    bound), and non-zero and within the precision's tolerance one ulp inside; the same holds for their weight rows."""
    got = _library_grads(conv, ei, ea, xs, gs)
    if p is not None:     # the bounds the library runs: Hardtanh's (lo, hi) as fp32 numbers, like the probed biases
        p = tuple(float(torch.tensor(v, dtype=torch.float32)) for v in p)
    ref = _reference_grads(conv, kind, p, ei, ea, xs, gs)
    n = _bound_biases(0.0, 1.0).numel()
    tol = 1e-4 if precision in ('fp32', 'f16x2') else 0.1
    for li in (4, 1):     # the second hidden layer's bias gradient, then its weight gradient (rows of the units)
        a = got[li][:n].double().cpu().reshape(n, -1)
        r = ref[li][:n].reshape(n, -1)
        sat = (r == 0).all(1)
        assert int(sat.sum()) == 4, (what, r)       # at, and beyond, each bound
        assert torch.equal((a == 0).all(1), sat), (what, li, a[:, 0], r[:, 0])
        assert rel_err(a[~sat], r[~sat]) < tol, (what, li, rel_err(a[~sat], r[~sat]))


BOUND_ACTS = [('relu6', None), ('hardtanh', (-0.3, 0.7))]


@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2'])
@pytest.mark.parametrize('kind,p', BOUND_ACTS)
def test_bound_probe_tensor_core_backward(kind, p, precision, formulation):
    from graph_pde_b200 import nn_conv
    formulation('off')
    ei, n = _hub_graph(e=6000, hub=2000)
    ea, xs, gs = _inputs(ei, n, T=1)
    conv = _bound_probe_conv(kind, p, precision)
    b0 = nn_conv.stats['mlp_backwards']
    _check_bound_units(conv, kind, p, ei, ea, xs, gs, precision, 'kept')
    assert nn_conv.stats['mlp_backwards'] > b0
    conv.zero_grad(set_to_none=True)
    conv.invalidate()
    old = nn_conv._KEEP_ACTS_MAX_BYTES
    nn_conv._KEEP_ACTS_MAX_BYTES = 0
    try:
        _check_bound_units(conv, kind, p, ei, ea, xs, gs, precision, 'recomputed')
    finally:
        nn_conv._KEEP_ACTS_MAX_BYTES = old


@pytest.mark.parametrize('precision', ['f16', 'f16x2'])
@pytest.mark.parametrize('kind,p', BOUND_ACTS)
def test_bound_probe_streamed_training(kind, p, precision, formulation):
    formulation('off')
    ei, n = _hub_graph()
    ea, xs, gs = _inputs(ei, n, T=1)
    h_bytes = 12032 * 128 * 2 * (2 if precision == 'f16x2' else 1)
    conv = _bound_probe_conv(kind, p, precision, edge_feature_bytes=h_bytes // 3, streamed_training=True)
    _check_bound_units(conv, kind, p, ei, ea, xs, gs, precision, 'streamed')


@pytest.mark.parametrize('precision', ['fp32', 'f16'])
@pytest.mark.parametrize('kind,p', BOUND_ACTS)
def test_bound_probe_cuda_core_backward(kind, p, precision, monkeypatch):
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_BWD_MODE', 'fp32')
    ei, n = _hub_graph(e=4000, hub=1000)
    ea, xs, gs = _inputs(ei, n, T=1)
    conv = _bound_probe_conv(kind, p, precision)
    _check_bound_units(conv, kind, p, ei, ea, xs, gs, 'fp32', 'cuda cores')


# ---- which kernels run -------------------------------------------------------------------------------------------------
_NAMES_SCRIPT = """
import sys, time, torch
sys.path.insert(0, %r)
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile
from graph_pde_b200 import nn_conv
from tests.test_gpu_edge_activation import _hub_graph, _inputs
from tests.test_gpu_edge_activation_more import _conv, ACTS
nn_conv._EDGE_KERNELS = 'off'
precision = sys.argv[1]
ei, n = _hub_graph(e=4000, hub=1000)
ea, (x,), (g,) = _inputs(ei, n)
ei, ea, x, g = ei.cuda(), ea.cuda().requires_grad_(), x.cuda().requires_grad_(), g.cuda()
for kind, p in ACTS:
    conv = _conv(kind, p, precision, 'mean')
    def step():
        conv.invalidate()
        (conv(x, ei, ea) * g).sum().backward()
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
    print('NAMES', kind, '|'.join(sorted(names)))
"""
_NAMES = {}


def _names(kind, precision):
    import os
    import subprocess
    import sys
    if precision not in _NAMES:
        root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
        res = subprocess.run([sys.executable, '-c', _NAMES_SCRIPT % root, precision], cwd=root,
                             stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
        assert res.returncode == 0, res.stdout
        _NAMES[precision] = {l.split(' ', 2)[1]: l.split(' ', 2)[2].split('|') for l in res.stdout.splitlines()
                             if l.startswith('NAMES ')}
    return _NAMES[precision][kind]


@pytest.mark.parametrize('precision', ['f16', 'f16x2', 'fp32'])
@pytest.mark.parametrize('kind,p', ACTS)
def test_activation_kernels_run(kind, p, precision):
    code = CODE[kind]
    names = _names(kind, precision)
    if precision == 'fp32':
        assert any(int(a[0]) == 8 + code for a in _template_args(names, 'k_sgemm_nt')), names
        assert any(int(a[0]) == code for a in _template_args(names, 'k_edge_layer1_act')), names
        assert any(int(a[0]) == code for a in _template_args(names, 'k_act_grad_colsum')), names
        assert not any('k_relu_mask_colsum' in nm for nm in names), names
    else:
        gemm = [int(a[3]) >> 3 for a in _template_args(names, 'k_gemm_tc')]
        assert code in gemm, names
        assert [int(a[2]) >> 1 for a in _template_args(names, 'k_dh')] == [code], names


# ---- CUDA-graph replay and fp16 range ---------------------------------------------------------------------------------
@pytest.mark.parametrize('precision', ['f16x2', 'f16'])
def test_graphed_train_step_with_selu(precision):
    import torch.nn.functional as F
    from graph_pde_b200 import GraphedTrainStep
    from graph_pde_b200.models import KernelNN
    from tests.test_gpu_graphed_train import TOL as RTOL, _assert_same, _cfg1_data, _clone_data, _eager_step

    def model():
        torch.manual_seed(0)
        m = KernelNN(32, 64, 3, 6, in_width=6, precision=precision)
        for i, layer in enumerate(m.conv1.nn.layers):
            if isinstance(layer, torch.nn.ReLU):
                m.conv1.nn.layers[i] = torch.nn.SELU()
        return m.to(DEV)
    d, y = _cfg1_data()
    mg, me = model(), model()
    me.load_state_dict(mg.state_dict())
    og = torch.optim.Adam(mg.parameters(), lr=1e-3, capturable=True)
    oe = torch.optim.Adam(me.parameters(), lr=1e-3, capturable=True)
    step = GraphedTrainStep(lambda d_, y_: F.mse_loss(mg(d_).view(-1), y_.view(-1)), mg, og, d, y)
    de = _clone_data(d)
    for k in range(3):
        loss_g = step.replay()
        loss_e = _eager_step(lambda d_, y_: F.mse_loss(me(d_).view(-1), y_.view(-1)), oe, de, y)
        _assert_same(loss_g, loss_e, mg, me, RTOL[precision], 'selu step %d' % k)


def test_graphed_forward_with_hardtanh():
    from graph_pde_b200 import GraphedForward
    ei, n = _hub_graph(e=4000, hub=1000)
    ea, (x, x2), _ = _inputs(ei, n, T=2)
    conv = _conv('hardtanh', (-0.3, 0.7), 'f16', 'mean')
    x, ei, ea = x.to(DEV), ei.to(DEV), ea.to(DEV)
    gf = GraphedForward(conv, x, ei, ea)
    x.copy_(x2.to(DEV))
    out = gf.replay().clone()
    with torch.no_grad():
        ref = conv(x2.to(DEV), ei, ea)
    assert rel_err(out, ref) < 1e-5


def test_fp16_overflow_is_reported_with_logsigmoid():
    """LogSigmoid is ~z for very negative z: a network whose pre-activations go below -65504 raises at f16 and runs at
    bf16; a non-finite edge attribute, which a clamp would map into the range, still counts."""
    ei, n = _hub_graph(e=4000, hub=1000)
    ea, (x,), _ = _inputs(ei, n)
    for precision in ('f16', 'bf16'):
        conv = _conv('logsigmoid', None, precision, 'mean')
        with torch.no_grad():
            conv.nn.layers[0].bias.fill_(-1e5)
        conv.invalidate()
        if precision == 'f16':
            with pytest.raises(FloatingPointError, match='edge-MLP activations left the fp16 range'), torch.no_grad():
                conv(x.to(DEV), ei.to(DEV), ea.to(DEV))
        else:
            with torch.no_grad():
                assert torch.isfinite(conv(x.to(DEV), ei.to(DEV), ea.to(DEV))).all()
    conv = _conv('relu6', None, 'f16', 'mean')
    bad = ea.clone()
    bad[7, 2] = float('inf')
    with pytest.raises(FloatingPointError, match='edge-MLP activations left the fp16 range'), torch.no_grad():
        conv(x.to(DEV), ei.to(DEV), bad.to(DEV))
