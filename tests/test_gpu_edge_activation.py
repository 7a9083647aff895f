"""Edge networks whose hidden activation is LeakyReLU, ELU, Tanh or Sigmoid, on the GPU: forward parity against the
fp64 restatement of tests/act_oracle.py on every application path and precision, gradients against fp64 autograd on
every backward path, one exact LeakyReLU(0.25) probe bit for bit, the kernels that run, and CUDA-graph replay and fp16
range reporting with these networks.  pytest -m gpu."""
import re
import subprocess
import sys

import pytest
import torch

from tests import act_oracle as A
from tests import act_probe as AP
from tests.helpers import TOL, rel_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ACTS = [('leaky_relu', 0.1), ('elu', 1.0), ('tanh', 0.0), ('sigmoid', 0.0)]
PRECS = ['f16', 'bf16', 'f16x2', 'fp32']
C = 64               # out = 64: the shape of the tensor-core backward and of the 16-bit diagonal-kernel build
DIMS = [6, 128, 128, C * C]
# gradients against fp64 autograd (DESIGN 5): tensor cores at f16 / bf16 8e-2 (edge_attr 0.3, and 5e-2 in the 2-norm);
# f16x2 and the CUDA-core backward 2e-4
GTOL = {'f16': 8e-2, 'bf16': 8e-2, 'f16x2': 2e-4, 'fp32': 2e-4}


def _mlp(dims, kind, p):
    from graph_pde_b200.models import DenseNet
    return DenseNet(dims, lambda: A.MODULES[kind](p))


def _hub_graph(n=400, e=12000, hub=6000, seed=0):
    """Source 0 has ``hub`` out-edges (the first half of the sorted edges: a prefix of a third of h ends inside it);
    nodes n-5.. have no in-edges."""
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n, (e,), generator=g)
    src[:hub] = 0
    dst = torch.randint(0, n - 5, (e,), generator=g)
    perm = torch.randperm(e, generator=g)
    return torch.stack([src[perm], dst[perm]]), n


def _low_degree_graph(n=3000, seed=1):
    """Two or three out-edges per source (formulation B territory)."""
    g = torch.Generator().manual_seed(seed)
    src = torch.arange(n).repeat_interleave(2 + (torch.arange(n) % 2))
    dst = torch.randint(0, n, (src.numel(),), generator=g)
    return torch.stack([src, dst]), n


def _inputs(ei, n, seed=0, T=1):
    g = torch.Generator().manual_seed(seed)
    ea = torch.randn(ei.size(1), DIMS[0], generator=g)
    xs = [torch.randn(n, C, generator=g) for _ in range(T)]
    gs = [torch.randn(n, C, generator=g) for _ in range(T)]
    return ea, xs, gs


def _conv(kind, p, precision, aggr='add', seed=0, cls=None, dims=DIMS, **kw):
    from graph_pde_b200.nn_conv import NNConv_old
    torch.manual_seed(seed)
    return (cls or NNConv_old)(C, C, _mlp(dims, kind, p), aggr=aggr, precision=precision, **kw).to(DEV)


def _params(conv):
    lin = [m for m in conv.nn.layers if isinstance(m, torch.nn.Linear)]
    return ([l.weight.detach().double().cpu() for l in lin], [l.bias.detach().double().cpu() for l in lin],
            conv.root.detach().double().cpu(), conv.bias.detach().double().cpu())


def _oracle_out(conv, kind, p, x, ei, ea, aggr, diag=False):
    ws, bs, root, bias = _params(conv)
    if diag:
        return A.diag_forward(x.double(), ei, ea.double(), ws, bs, root, bias, aggr, kind, p)
    return A.nnconv_forward(x.double(), ei, ea.double(), ws, bs, root, bias, aggr, kind, p)[0]


@pytest.fixture
def formulation(monkeypatch):
    from graph_pde_b200 import nn_conv

    def set_(mode):
        monkeypatch.setattr(nn_conv, '_EDGE_KERNELS', mode)
    return set_


# ---- forward parity ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('aggr', ['add', 'mean', 'max'])
@pytest.mark.parametrize('precision', PRECS)
@pytest.mark.parametrize('kind,p', ACTS)
def test_forward_cached(kind, p, precision, aggr, formulation):
    """Formulation C over the whole cached h."""
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
    """A resident prefix of a third of h ends inside source 0's 6000 out-edges; every application recomputes the rest
    chunk by chunk.  The cached run's result up to the order of the fp32 scatter additions (DESIGN 5: 1e-5)."""
    from graph_pde_b200 import nn_conv
    formulation('off')
    ei, n = _hub_graph()
    ea, (x,), _ = _inputs(ei, n)
    conv = _conv(kind, p, precision, 'mean')
    with torch.no_grad():
        cached = conv(x.to(DEV), ei.to(DEV), ea.to(DEV))
    h_bytes = 12032 * 128 * 2 * (2 if precision == 'f16x2' else 1)
    conv.edge_feature_bytes = h_bytes // 3
    conv.invalidate()
    s0 = nn_conv.stats['streamed_chunk_passes']
    with torch.no_grad():
        out = conv(x.to(DEV), ei.to(DEV), ea.to(DEV))
    assert nn_conv.stats['streamed_chunk_passes'] > s0
    ef = next(iter(conv._h_cache.values()))
    assert 0 < ef.E_res < 6000, ef.E_res
    assert rel_err(out, cached) < 1e-5
    assert rel_err(out, _oracle_out(conv, kind, p, x, ei, ea, 'mean')) < TOL[precision]


@pytest.mark.parametrize('precision', ['f16', 'bf16'])
@pytest.mark.parametrize('kind,p', ACTS)
def test_forward_formulation_b(kind, p, precision, formulation):
    """Per-edge kernel matrices on a graph of two or three out-edges per source."""
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


# ---- gradients ---------------------------------------------------------------------------------------------------------
def _reference_grads(conv, kind, p, ei, ea, xs, gs, diag=False):
    ws, bs, root, bias = _params(conv)
    leaves = [w.requires_grad_() for w in ws] + [b.requires_grad_() for b in bs] + [root.requires_grad_(),
                                                                                   bias.requires_grad_()]
    ea64 = ea.double().requires_grad_()
    x64 = [x.double().requires_grad_() for x in xs]
    loss = 0
    for x, g in zip(x64, gs):
        if diag:
            out = A.diag_forward(x, ei, ea64, ws, bs, root, bias, conv.aggr, kind, p)
        else:
            out = A.nnconv_forward(x, ei, ea64, ws, bs, root, bias, conv.aggr, kind, p)[0]
        loss = loss + (out * g.double()).sum()
    loss.backward()
    return [l.grad for l in leaves] + [ea64.grad] + [x.grad for x in x64]


def _library_grads(conv, ei, ea, xs, gs):
    ea_d = ea.to(DEV).requires_grad_()
    x_d = [x.to(DEV).requires_grad_() for x in xs]
    loss = 0
    for x, g in zip(x_d, gs):
        loss = loss + (conv(x, ei.to(DEV), ea_d) * g.to(DEV)).sum()
    loss.backward()
    lin = [m for m in conv.nn.layers if isinstance(m, torch.nn.Linear)]
    return ([l.weight.grad for l in lin] + [l.bias.grad for l in lin] + [conv.root.grad, conv.bias.grad] +
            [ea_d.grad] + [x.grad for x in x_d])


def _ea_index(conv):
    return 2 * len([m for m in conv.nn.layers if isinstance(m, torch.nn.Linear)]) + 2


def _check_grads(conv, kind, p, ei, ea, xs, gs, precision, what, diag=False):
    got = _library_grads(conv, ei, ea, xs, gs)
    ref = _reference_grads(conv, kind, p, ei, ea, xs, gs, diag)
    k_ea = _ea_index(conv)
    for i, (a, b) in enumerate(zip(got, ref)):
        err = rel_err(a, b)
        tol = 0.3 if (i == k_ea and precision in ('f16', 'bf16')) else GTOL[precision]
        assert err < tol, (what, i, err)
        if i == k_ea and precision in ('f16', 'bf16'):
            d = a.detach().double().cpu() - b
            assert float(d.norm() / b.norm()) < 5e-2, (what, 'edge_attr 2-norm', float(d.norm() / b.norm()))
    return got


@pytest.mark.parametrize('T', [1, 6])
@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2'])
@pytest.mark.parametrize('kind,p', ACTS)
def test_tensor_core_backward(kind, p, precision, T, formulation):
    """T applications of one conv, kept activations (the default) and recomputed ones: both against fp64 autograd, and
    bit for bit against each other."""
    from graph_pde_b200 import nn_conv
    formulation('off')
    ei, n = _hub_graph(e=6000, hub=2000)
    ea, xs, gs = _inputs(ei, n, T=T)
    conv = _conv(kind, p, precision, 'mean')
    b0 = nn_conv.stats['mlp_backwards']
    kept = _check_grads(conv, kind, p, ei, ea, xs, gs, precision, 'kept')
    assert nn_conv.stats['mlp_backwards'] > b0            # the tensor-core backward ran
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
    """Training on streamed edge features (a third of h resident): the backward recomputes the streamed activations."""
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
    """The fp32 CUDA-core backward (precision 'fp32', or NNCONV_B200_BACKWARD=fp32 under an f16 forward)."""
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_BWD_MODE', 'fp32')
    ei, n = _hub_graph(e=4000, hub=1000)
    ea, xs, gs = _inputs(ei, n, T=2)
    conv = _conv(kind, p, precision, 'mean')
    _check_grads(conv, kind, p, ei, ea, xs, gs, 'fp32', 'cuda cores')


@pytest.mark.parametrize('precision', ['f16', 'fp32'])
@pytest.mark.parametrize('kind,p', ACTS)
def test_diag_backward(kind, p, precision):
    """DiagNNConv's fp32 backward through recomputed activations (3e-2 at f16, whose d carries the 16-bit h)."""
    from graph_pde_b200.nn_conv import DiagNNConv
    ei, n = _hub_graph(e=4000, hub=1000)
    ea, xs, gs = _inputs(ei, n, T=2)
    conv = _conv(kind, p, precision, 'add', cls=DiagNNConv, dims=[6, 128, 128, C])
    got = _library_grads(conv, ei, ea, xs, gs)
    ref = _reference_grads(conv, kind, p, ei, ea, xs, gs, diag=True)
    for i, (a, b) in enumerate(zip(got, ref)):
        assert rel_err(a, b) < (3e-2 if precision == 'f16' else 1e-4), (i, rel_err(a, b))


# ---- exact LeakyReLU(0.25) probe ---------------------------------------------------------------------------------------
def _probe_conv(pr, precision):
    from graph_pde_b200.nn_conv import NNConv_old
    mlp = _mlp(pr.layers, 'leaky_relu', AP.SLOPE)
    conv = NNConv_old(pr.cin, pr.cout, mlp, aggr='add', precision=precision)
    with torch.no_grad():
        for l, w, b in zip([m for m in mlp.layers if isinstance(m, torch.nn.Linear)], pr.ws, pr.bs):
            l.weight.copy_(w)
            l.bias.copy_(b)
        conv.root.copy_(pr.root)
        conv.bias.copy_(pr.bias)
    return conv.to(DEV)


@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2', 'fp32'])
def test_exact_leaky_relu_probe(precision, formulation):
    """Pre-activations of both signs, T = 2: the output of every application and every gradient (x, each weight and
    bias, root, bias, edge_attr row by row) equal fp64 autograd bit for bit (the budget is proved on the CPU)."""
    formulation('off')
    ei, n = AP.graph()
    pr = AP.make(ei, n, precision=precision)
    conv = _probe_conv(pr, precision)
    ea = pr.ea.float()
    with torch.no_grad():
        for x in pr.x:
            out = conv(x.float().to(DEV), ei.to(DEV), ea.to(DEV))
            ref = A.nnconv_forward(x, ei, pr.ea.double(), pr.ws, pr.bs, pr.root, pr.bias, 'add', 'leaky_relu',
                                   AP.SLOPE)[0]
            assert torch.equal(out.double().cpu(), ref)
    conv.invalidate()
    from graph_pde_b200 import nn_conv
    b0 = nn_conv.stats['mlp_backwards']
    got = _library_grads(conv, ei, ea, [x.float() for x in pr.x], [g.float() for g in pr.grad_out])
    assert (nn_conv.stats['mlp_backwards'] > b0) == (precision != 'fp32')     # tensor cores at 16 bits
    ref = _reference_grads(conv, 'leaky_relu', AP.SLOPE, ei, ea, pr.x, pr.grad_out)
    for i, (a, b) in enumerate(zip(got, ref)):
        assert torch.equal(a.double().cpu(), b), (i, float((a.double().cpu() - b).abs().max()))


# ---- which kernels run -------------------------------------------------------------------------------------------------
_NAMES_SCRIPT = """
import sys, time, torch
sys.path.insert(0, %r)
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile
from graph_pde_b200 import nn_conv
from tests.test_gpu_edge_activation import _conv, _hub_graph, _inputs, ACTS
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


def _kernel_names(kind, precision):
    """Kernels one forward + backward of each activation launches at ``precision``, profiled in a fresh process (the
    profiler state of the test process is left alone)."""
    import os
    if precision not in _NAMES:
        root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
        res = subprocess.run([sys.executable, '-c', _NAMES_SCRIPT % root, precision], cwd=root,
                             stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
        assert res.returncode == 0, res.stdout
        _NAMES[precision] = {l.split(' ', 2)[1]: l.split(' ', 2)[2].split('|') for l in res.stdout.splitlines()
                             if l.startswith('NAMES ')}
    assert kind in _NAMES[precision], _NAMES[precision]
    return _NAMES[precision][kind]


def _template_args(names, kernel):
    out = []
    for nm in names:
        m = re.search(r'\b%s<([^>]*)>' % kernel, nm)
        if m:
            out.append([a.strip() for a in m.group(1).split(',')])
    return out


@pytest.mark.parametrize('precision', ['f16', 'f16x2', 'fp32'])
@pytest.mark.parametrize('kind,p', ACTS)
def test_activation_kernels_run(kind, p, precision):
    """The activation is fused where ReLU is: the tensor-core GEMMs run the epilogues of this activation (EPI >> 3) and
    k_dh its derivative (MODE >> 1) at 16 bits; fp32 runs the CUDA-core first layer, GEMM and backward of it."""
    code = {'leaky_relu': 1, 'elu': 2, 'tanh': 3, 'sigmoid': 4}[kind]
    names = _kernel_names(kind, precision)
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
def test_graphed_train_step_with_tanh(precision):
    """GraphedTrainStep replays of a KernelNN whose edge network runs Tanh equal the same steps taken eagerly."""
    import torch.nn.functional as F
    from graph_pde_b200 import GraphedTrainStep
    from graph_pde_b200.models import KernelNN
    from tests.test_gpu_graphed_train import TOL as RTOL, _assert_same, _cfg1_data, _clone_data, _eager_step

    def model():
        torch.manual_seed(0)
        m = KernelNN(32, 64, 3, 6, in_width=6, precision=precision)
        for i, layer in enumerate(m.conv1.nn.layers):
            if isinstance(layer, torch.nn.ReLU):
                m.conv1.nn.layers[i] = torch.nn.Tanh()
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
        _assert_same(loss_g, loss_e, mg, me, RTOL[precision], 'tanh step %d' % k)


@pytest.mark.parametrize('kind,p', ACTS)
def test_graphed_forward_replays(kind, p):
    """A GraphedForward of a conv with the activation replays the eager forward of new inputs (up to the order of the
    fp32 scatter additions)."""
    from graph_pde_b200 import GraphedForward
    ei, n = _hub_graph(e=4000, hub=1000)
    ea, (x, x2), _ = _inputs(ei, n, T=2)
    conv = _conv(kind, p, 'f16', 'mean')
    x, ei, ea = x.to(DEV), ei.to(DEV), ea.to(DEV)
    gf = GraphedForward(conv, x, ei, ea)
    x.copy_(x2.to(DEV))
    out = gf.replay().clone()
    with torch.no_grad():
        ref = conv(x2.to(DEV), ei, ea)
    assert rel_err(out, ref) < 1e-5


def test_fp16_overflow_is_reported_with_elu():
    """An ELU network whose activations leave the fp16 range raises at f16 and runs at bf16; a non-finite edge
    attribute, which Tanh would map into the range, still counts."""
    ei, n = _hub_graph(e=4000, hub=1000)
    ea, (x,), _ = _inputs(ei, n)
    for precision in ('f16', 'bf16'):
        conv = _conv('elu', 1.0, precision, 'mean')
        with torch.no_grad():
            for m in conv.nn.layers:
                if isinstance(m, torch.nn.Linear):
                    m.weight.mul_(1024.0)
        conv.invalidate()
        if precision == 'f16':
            with pytest.raises(FloatingPointError, match='edge-MLP activations left the fp16 range'), torch.no_grad():
                conv(x.to(DEV), ei.to(DEV), ea.to(DEV))
        else:
            with torch.no_grad():
                assert torch.isfinite(conv(x.to(DEV), ei.to(DEV), ea.to(DEV))).all()
    conv = _conv('tanh', 0.0, 'f16', 'mean')
    bad = ea.clone()
    bad[7, 2] = float('inf')
    with pytest.raises(FloatingPointError, match='edge-MLP activations left the fp16 range'), torch.no_grad():
        conv(x.to(DEV), ei.to(DEV), bad.to(DEV))
