"""GPU: gradients w.r.t. edge_attr (nnconv_backward_mlp_ex on the tensor cores, nnconv_backward_ex on the CUDA cores)
against autograd through the oracle with edge_attr as a leaf -- single convs, the autograd interface, an inverse problem
through KernelNN (theta -> node features and edge attributes) and the orthogonal MGKN hierarchy.  Errors are
max|g - ref| / max|ref| per tensor.  pytest -m gpu."""
import numpy as np
import pytest
import torch

from oracle import nnconv_oracle as O
from tests.helpers import DenseNetLike, emulated_nnconv_forward, make_conv

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
GTOL = {'f16': 3e-3, 'bf16': 3e-2}       # vs autograd through the forward that rounds where the kernels round
GTOL_EXACT = 8e-2                        # vs the exact fp64 oracle (16-bit operands), gradients summed over edges
# edge_attr's gradient vs the exact fp64 oracle.  It is a PER-EDGE quantity: a ReLU unit of one edge that the 16-bit
# forward flips (tests/helpers.py) changes that edge's row by ~1/sqrt(width) of its size, and no sum over edges averages
# the flip out as it does for the parameter gradients -- the max-norm error is that of the worst edge (0.09 .. 0.16 in
# the cases below on the H100, while the rounding-consistent reference agrees to < 1e-3 at f16).  The exact oracle is
# therefore a loose bound in the max norm plus a bound on the relative 2-norm error, which the few flipped rows barely
# move; the tight check is GTOL against the rounding-consistent reference.
GTOL_EXACT_EA = 0.3
GTOL_EXACT_EA_L2 = 5e-2
FP32_TOL = 2e-4                          # CUDA-core backward vs the exact fp64 oracle


def _relerr(got, ref):
    ref = ref.detach().double().cpu()
    return float((got.detach().double().cpu() - ref).abs().max() / ref.abs().max().clamp(min=1e-30))


def _relerr_l2(got, ref):
    ref = ref.detach().double().cpu()
    return float((got.detach().double().cpu() - ref).norm() / ref.norm().clamp(min=1e-30))


def _exact_ea_ok(got, ref):
    return _relerr(got, ref) < GTOL_EXACT_EA and _relerr_l2(got, ref) < GTOL_EXACT_EA_L2


def _graph(gen, N, E, hub=False):
    src = torch.randint(0, N - 5, (E,), generator=gen)
    dst = torch.randint(2, N, (E,), generator=gen)
    if hub:
        src[:300] = 3
    order = torch.argsort(src, stable=True) if not hub else torch.arange(E)
    return torch.stack([src[order], dst[order]])


def _problem(layers, cin, cout, rw, bs, N, E, gscale=1.0):
    gen = torch.Generator().manual_seed(17)
    ei = _graph(gen, N, E, hub=True)                 # unsorted sources + a hub with several tiles: exercises perm
    ea = torch.randn(E, layers[0], generator=gen)
    x = torch.randn(N, cin, generator=gen)
    torch.manual_seed(3)
    lin = [m for m in DenseNetLike(layers).layers if isinstance(m, torch.nn.Linear)]
    ws = [l.weight.detach().clone() for l in lin]
    bsl = [l.bias.detach().clone() for l in lin]
    root = torch.randn(cin, cout) * 0.2 if rw else None
    bias = torch.randn(cout) * 0.2 if bs else None
    gout = torch.randn(N, cout, generator=gen) * gscale
    return ei, ea, x, ws, bsl, root, bias, gout


def _reference(fwd, x, ea, ws, bsl, root, bias, gout):
    """autograd (fp64, CPU) of sum(fwd(...) * gout) w.r.t. x, edge_attr and every parameter"""
    lv = {'x': x.double(), 'ea': ea.double()}
    for i in range(len(ws)):
        lv['W%d' % i], lv['b%d' % i] = ws[i].double(), bsl[i].double()
    if root is not None:
        lv['root'] = root.double()
    if bias is not None:
        lv['bias'] = bias.double()
    lv = {k: v.requires_grad_(True) for k, v in lv.items()}
    wr = [lv['W%d' % i] for i in range(len(ws))]
    br = [lv['b%d' % i] for i in range(len(ws))]
    (fwd(lv['x'], lv['ea'], wr, br, lv.get('root'), lv.get('bias')) * gout.double()).sum().backward()
    return {k: v.grad for k, v in lv.items()}


def _run(conv, x, ei, ea, gout, ea_grad):
    xd = x.to(DEV).requires_grad_(True)
    ead = ea.to(DEV).requires_grad_(ea_grad)
    out = conv(xd, ei.to(DEV), ead)
    (out * gout.to(DEV)).sum().backward()
    got = {'x': xd.grad}
    for i, l in enumerate([m for m in conv.nn.layers if isinstance(m, torch.nn.Linear)]):
        got['W%d' % i], got['b%d' % i] = l.weight.grad, l.bias.grad
    if conv.root is not None:
        got['root'] = conv.root.grad
    if conv.bias is not None:
        got['bias'] = conv.bias.grad
    if ea_grad:
        got['ea'] = ead.grad
    return got


TC_CASES = [       # the cases of test_gpu_backward_tc.test_tc_backward_matches_autograd_through_oracle
    ([6, 64, 64, 64 * 64], 64, 'mean', True, True, 'f16'),
    ([6, 64, 64, 64 * 64], 64, 'add', True, True, 'bf16'),
    ([6, 128, 32 * 64], 32, 'mean', False, False, 'f16'),            # 2-layer MLP: dz_1 comes out of k_dh
    ([4, 256, 320, 64 * 64], 64, 'mean', True, False, 'f16'),        # k_in = 4, Kp = 320
    ([6, 16, 32, 24, 64 * 64], 64, 'add', False, True, 'f16'),       # 4-layer MLP, widths padded to 64
]


@pytest.mark.parametrize('layers,cin,aggr,rw,bs,prec', TC_CASES)
def test_tc_edge_attr_grad_matches_autograd(layers, cin, aggr, rw, bs, prec, monkeypatch):
    """Tensor-core path, with kept and with recomputed hidden activations and with a workspace small enough for
    several source batches: edge_attr's gradient against the rounding-consistent and the exact reference, one
    tensor-core MLP pass, and every other gradient as in a run where edge_attr needs none."""
    from graph_pde_b200 import nn_conv
    from graph_pde_b200.nn_conv import NNConv_old, stats
    cout = 64
    ei, ea, x, ws, bsl, root, bias, gout = _problem(layers, cin, cout, rw, bs, 150, 2500, gscale=1e-3)
    ref_exact = _reference(lambda xr, er, wr, br, rr, bbr: O.nnconv_forward(xr, ei, er, wr, br, rr, bbr, aggr, cin, cout),
                           x, ea, ws, bsl, root, bias, gout)
    ref_emul = _reference(lambda xr, er, wr, br, rr, bbr: emulated_nnconv_forward(xr, ei, er, wr, br, rr, bbr, aggr, prec),
                          x, ea, ws, bsl, root, bias, gout)
    report, ok = [], True
    for cfg in ('kept activations', 'recomputed activations', 'one source group per batch'):
        monkeypatch.setattr(nn_conv, '_KEEP_ACTS_MAX_BYTES', 0 if cfg == 'recomputed activations' else 64 << 30)
        monkeypatch.setattr(nn_conv, '_BWD_MLP_WS_BYTES', 1 if cfg == 'one source group per batch' else 4 << 30)
        base = _run(make_conv(NNConv_old, ws, bsl, root, bias, aggr, cin, cout, prec, DEV), x, ei, ea, gout, False)
        n0 = stats.get('mlp_backwards', 0)
        got = _run(make_conv(NNConv_old, ws, bsl, root, bias, aggr, cin, cout, prec, DEV), x, ei, ea, gout, True)
        assert stats.get('mlp_backwards', 0) == n0 + 1          # the tensor-core pass ran, once
        assert got['ea'].shape == ea.shape and got['ea'].dtype == ea.dtype
        e = dict(emul=_relerr(got['ea'], ref_emul['ea']), exact=_relerr(got['ea'], ref_exact['ea']),
                 exact_l2=_relerr_l2(got['ea'], ref_exact['ea']),
                 others=max(_relerr(got[k], base[k]) for k in base))
        report.append((cfg, e))
        ok = ok and e['emul'] < GTOL[prec] and _exact_ea_ok(got['ea'], ref_exact['ea']) and e['others'] < GTOL[prec]
    print(report)
    assert ok, report


def test_tc_edge_attr_grad_sums_applications():
    """One conv applied T = 7 times (the MLP pass runs in two groups of applications): one summed gradient."""
    from graph_pde_b200.nn_conv import NNConv_old, stats
    layers, cin, cout, aggr, prec, T = [6, 64, 64, 64 * 64], 64, 64, 'mean', 'f16', 7
    ei, ea, _, ws, bsl, root, bias, _ = _problem(layers, cin, cout, True, True, 150, 2500)
    gen = torch.Generator().manual_seed(29)
    xs = [torch.randn(150, cin, generator=gen) for _ in range(T)]
    gouts = [torch.randn(150, cout, generator=gen) * 1e-2 for _ in range(T)]

    def ref(fwd):
        er = ea.double().requires_grad_(True)
        sum((fwd(x.double(), er) * g.double()).sum() for x, g in zip(xs, gouts)).backward()
        return er.grad
    wd, bd = [w.double() for w in ws], [b.double() for b in bsl]
    ref_exact = ref(lambda xr, er: O.nnconv_forward(xr, ei, er, wd, bd, root.double(), bias.double(), aggr, cin, cout))
    ref_emul = ref(lambda xr, er: emulated_nnconv_forward(xr, ei, er, wd, bd, root.double(), bias.double(), aggr, prec))
    conv = make_conv(NNConv_old, ws, bsl, root, bias, aggr, cin, cout, prec, DEV)
    ead = ea.to(DEV).requires_grad_(True)
    eid = ei.to(DEV)
    n0 = stats.get('mlp_backwards', 0)
    loss = sum((conv(x.to(DEV), eid, ead) * g.to(DEV)).sum() for x, g in zip(xs, gouts))
    loss.backward()
    assert stats.get('mlp_backwards', 0) == n0 + 1
    e = (_relerr(ead.grad, ref_emul), _relerr(ead.grad, ref_exact), _relerr_l2(ead.grad, ref_exact))
    assert e[0] < GTOL[prec] and _exact_ea_ok(ead.grad, ref_exact), e


@pytest.mark.parametrize('layers,cin,cout,aggr,rw,bs,fwd_prec', [
    ([6, 32, 48, 16 * 16], 16, 16, 'mean', True, True, 'fp32'),
    ([6, 64, 64, 32 * 32], 32, 32, 'mean', True, True, 'f16'),      # tensor-core forward, fp32 backward
    ([4, 24, 5 * 7], 5, 7, 'add', False, True, 'fp32'),             # 2-layer MLP, odd shapes, no root
    ([3, 8 * 8], 8, 8, 'mean', True, False, 'fp32'),                # single Linear edge network: dh[:, :k_in]
    ([6, 16, 32, 24, 64 * 64], 64, 64, 'mean', False, False, 'f16'),  # 4-layer MLP, MGKN style
    ([6, 64, 64, 32 * 32], 32, 32, 'add', True, True, 'f16x2'),
])
def test_fp32_edge_attr_grad_matches_oracle(layers, cin, cout, aggr, rw, bs, fwd_prec, monkeypatch):
    from graph_pde_b200 import nn_conv
    from graph_pde_b200.nn_conv import NNConv_old
    monkeypatch.setattr(nn_conv, '_BWD_MODE', 'fp32')
    ei, ea, x, ws, bsl, root, bias, gout = _problem(layers, cin, cout, rw, bs, 120, 1500)
    ref = _reference(lambda xr, er, wr, br, rr, bbr: O.nnconv_forward(xr, ei, er, wr, br, rr, bbr, aggr, cin, cout),
                     x, ea, ws, bsl, root, bias, gout)
    got = _run(make_conv(NNConv_old, ws, bsl, root, bias, aggr, cin, cout, fwd_prec, DEV), x, ei, ea, gout, True)
    errs = {k: _relerr(got[k], ref[k]) for k in got}
    assert all(v < FP32_TOL for v in errs.values()), errs


@pytest.mark.parametrize('mode', ['auto', 'fp32'])
def test_only_edge_attr_requires_grad(mode, monkeypatch):
    """A frozen model and an x without gradient (an inverse loop): the output still carries a grad_fn and edge_attr
    gets its gradient."""
    from graph_pde_b200 import nn_conv
    from graph_pde_b200.nn_conv import NNConv_old
    monkeypatch.setattr(nn_conv, '_BWD_MODE', mode)
    layers, cin, cout, aggr = [6, 64, 64, 64 * 64], 64, 64, 'mean'
    ei, ea, x, ws, bsl, root, bias, gout = _problem(layers, cin, cout, True, True, 150, 2500)
    conv = make_conv(NNConv_old, ws, bsl, root, bias, aggr, cin, cout, 'f16', DEV)
    conv.requires_grad_(False)
    ead = ea.to(DEV).requires_grad_(True)
    out = conv(x.to(DEV), ei.to(DEV), ead)
    assert out.grad_fn is not None
    (out * gout.to(DEV)).sum().backward()
    fwd = emulated_nnconv_forward if mode == 'auto' else (lambda *a: O.nnconv_forward(*a[:8], cin, cout))
    er = ea.double().requires_grad_(True)
    (fwd(x.double(), ei, er, [w.double() for w in ws], [b.double() for b in bsl], root.double(), bias.double(), aggr,
         'f16') * gout.double()).sum().backward()
    assert _relerr(ead.grad, er.grad) < (GTOL['f16'] if mode == 'auto' else FP32_TOL)
    assert all(p.grad is None for p in conv.parameters())


@pytest.mark.parametrize('mode', ['auto', 'fp32'])
def test_edge_attr_grad_shape_and_dtype(mode, monkeypatch):
    """1-D edge_attr gets a 1-D gradient, float64 edge_attr a float64 one."""
    from graph_pde_b200 import nn_conv
    from graph_pde_b200.nn_conv import NNConv_old
    monkeypatch.setattr(nn_conv, '_BWD_MODE', mode)
    prec = 'f16' if mode == 'auto' else 'fp32'
    cin = cout = 64
    for layers, one_d, dt in (([1, 64, 64 * 64], True, torch.float32), ([6, 64, 64, 64 * 64], False, torch.float64)):
        ei, ea, x, ws, bsl, root, bias, gout = _problem(layers, cin, cout, True, True, 150, 2500)
        ea = (ea[:, 0] if one_d else ea).to(dt)
        ead = ea.to(DEV).requires_grad_(True)
        conv = make_conv(NNConv_old, ws, bsl, root, bias, 'mean', cin, cout, prec, DEV)
        (conv(x.to(DEV), ei.to(DEV), ead) * gout.to(DEV)).sum().backward()
        assert ead.grad.shape == ea.shape and ead.grad.dtype == dt
        er = ea.double().requires_grad_(True)
        wd, bd = [w.double() for w in ws], [b.double() for b in bsl]
        er2 = er.unsqueeze(-1) if one_d else er
        if mode == 'auto':      # tensor-core path: the rounding-consistent reference
            out = emulated_nnconv_forward(x.double(), ei, er2, wd, bd, root.double(), bias.double(), 'mean', prec)
        else:
            out = O.nnconv_forward(x.double(), ei, er2, wd, bd, root.double(), bias.double(), 'mean', cin, cout)
        (out * gout.double()).sum().backward()
        assert _relerr(ead.grad, er.grad) < (GTOL[prec] if mode == 'auto' else FP32_TOL), (layers, dt)


@pytest.mark.parametrize('mode', ['auto', 'fp32'])
def test_empty_graph_gives_empty_gradient(mode, monkeypatch):
    from graph_pde_b200 import nn_conv
    from graph_pde_b200.nn_conv import NNConv_old
    monkeypatch.setattr(nn_conv, '_BWD_MODE', mode)
    torch.manual_seed(0)
    conv = NNConv_old(64, 64, DenseNetLike([6, 64, 64 * 64]), aggr='mean', precision='f16').to(DEV)
    x = torch.randn(20, 64, device=DEV, requires_grad=True)
    ead = torch.zeros(0, 6, device=DEV, requires_grad=True)
    out = conv(x, torch.zeros(2, 0, dtype=torch.int64, device=DEV), ead)
    out.sum().backward()
    assert ead.grad is not None and ead.grad.shape == (0, 6)
    assert torch.allclose(x.grad, torch.ones(20, 64, device=DEV) @ conv.root.detach().t(), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize('precision', ['fp32', 'f16'])
def test_kernelnn_inverse_problem_gradient(precision):
    """d loss / d theta through KernelNN, theta entering the node features and the edge attributes
    (graphs.ball_edge_attr, differentiable): the coefficient-recovery gradient of an inverse problem."""
    from graph_pde_b200 import graphs
    from graph_pde_b200.models import KernelNN
    s, r, w, kw, T = 12, 0.3, 64, 128, 3
    gen = torch.Generator().manual_seed(7)
    ei = graphs.ball_connectivity(s, r)
    grid = graphs.square_grid(s, dtype=torch.float64)
    theta0 = torch.randn(s * s, generator=gen, dtype=torch.float64)
    feats = torch.randn(s * s, 3, generator=gen, dtype=torch.float64)
    y = torch.randn(s * s, 1, generator=gen, dtype=torch.float64)
    torch.manual_seed(0)
    model = KernelNN(w, kw, T, 6, in_width=6, precision=precision).to(DEV)
    model.requires_grad_(False)

    def inputs(theta, g, f):
        x = torch.cat([g, theta[:, None], f], dim=1)
        src, dst = ei[0].to(theta.device), ei[1].to(theta.device)
        ea = torch.cat([g[src], g[dst], theta[src, None], theta[dst, None]], dim=1)
        return x, ea

    class D(object):
        pass
    theta = theta0.float().to(DEV).requires_grad_(True)
    d = D()
    d.x = torch.cat([grid.float().to(DEV), theta[:, None], feats.float().to(DEV)], dim=1)
    d.edge_index = ei.to(DEV)
    d.edge_attr = graphs.ball_edge_attr(grid.float().to(DEV), d.edge_index, theta)
    conv_outs = []
    hook = model.conv1.register_forward_hook(lambda m, i, o: conv_outs.append(o.detach().double().cpu()))
    torch.nn.functional.mse_loss(model(d), y.float().to(DEV)).backward()
    hook.remove()
    st = {k: v.detach().cpu().double() for k, v in model.state_dict().items()}

    def ref_grad(emulated):
        th = theta0.clone().requires_grad_(True)
        x, ea = inputs(th, grid, feats)
        if not emulated:
            out = O.kernelnn_forward(x, ei, ea, st, T)
        else:      # mask-consistent: node ReLUs evaluated at the CUDA path's own conv outputs
            ws, bs = O.mlp_params_from_state(st, 'conv1.nn.')
            h = torch.nn.functional.linear(x, st['fc1.weight'], st['fc1.bias'])
            for k in range(T):
                o = emulated_nnconv_forward(h, ei, ea, ws, bs, st['conv1.root'], st['conv1.bias'], 'mean', precision)
                h = torch.relu(o + (conv_outs[k] - o).detach())
            out = torch.nn.functional.linear(h, st['fc2.weight'], st['fc2.bias'])
        torch.nn.functional.mse_loss(out, y).backward()
        return th.grad
    if precision == 'fp32':
        e = _relerr(theta.grad, ref_grad(False))
        print('theta.grad error (fp32):', e)
        assert e < 5e-4
    else:
        e_emul, e_exact = _relerr(theta.grad, ref_grad(True)), _relerr(theta.grad, ref_grad(False))
        print('theta.grad error (f16): rounding-consistent %.3g, exact %.3g' % (e_emul, e_exact))
        assert e_emul < GTOL['f16'] and e_exact < GTOL_EXACT, (e_emul, e_exact)


@pytest.mark.usefixtures('edge_kernel_mode')
@pytest.mark.parametrize('precision', ['fp32', 'f16'])
def test_mgkn_orthogonal_edge_attr_grads(precision):
    """Orthogonal 1-D MGKN (width 64: the tensor-core backward at 16 bit) with leaf edge_attr_list tensors, against
    autograd through oracle.mgkn_orthogonal_forward."""
    from graph_pde_b200 import graphs
    from graph_pde_b200.models import MGKN
    s, w, kw, depth = 64, 64, 64, 1
    theta = torch.randn(s, generator=torch.Generator().manual_seed(11))
    X, eis, eas = graphs.multi_pole_grid1d(theta, s)
    torch.manual_seed(0)
    model = MGKN(width=w, ker_width=kw, depth=depth, ker_in=4, in_width=2, s=s, precision=precision).to(DEV)
    gout = torch.randn(s, 1, generator=torch.Generator().manual_seed(12))
    ead = [e.to(DEV).requires_grad_(True) for e in eas]
    out = model(([x.to(DEV) for x in X], None, [e.to(DEV) for e in eis], ead))
    (out * gout.to(DEV)).sum().backward()
    st = {k: v.detach().cpu().double() for k, v in model.state_dict().items()}
    er = [e.double().requires_grad_(True) for e in eas]
    (O.mgkn_orthogonal_forward(X[0].double(), eis, er, st, depth, w, s) * gout.double()).sum().backward()
    errs = [_relerr(a.grad, b.grad) for a, b in zip(ead, er)]
    print('MGKN edge_attr_list gradient errors (%s):' % precision, errs)
    assert max(errs) < (5e-4 if precision == 'fp32' else GTOL_EXACT), errs
