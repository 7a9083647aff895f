"""aggr='mean' bit for bit on exact probes whose every in-degree is a power of two (tests/probes.py, MEAN_FORWARD and
MEAN_BACKWARD): inv_deg = 1/deg is then exact, each message or gradient row times inv_deg only shifts an exponent, and
the library must equal the fp64 mean (the oracle, or autograd through it) at every node and every gradient row, on every
forward path, schedule and backward.  A 1/deg off by one ulp, a degree read at the wrong end of an edge, or a G that
misses its scale fails here where a tolerance would not."""
import pytest
import torch

from tests import probes as P
from tests.test_gpu_exact_backward import _library, _reference as _grad_reference, assert_grads_equal, hub_edges
from tests.test_gpu_exact_forward import PATHS, SPLIT_PATHS, _h_bytes, _reference as _fwd_reference

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
MF, MB = P.MEAN_FORWARD, P.MEAN_BACKWARD


@pytest.fixture
def lib_options():
    from graph_pde_b200 import _lib
    touched = []

    def setter(name, value):
        touched.append(name)
        _lib.set_option(name, value)
    yield setter
    for name in touched:
        _lib.set_option(name, None)


@pytest.fixture(autouse=True)
def formulation_c(monkeypatch):
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_EDGE_KERNELS', 'off')


def _cls():
    from graph_pde_b200.nn_conv import NNConv_old
    return NNConv_old


def _probe(table, name, precision):
    p = P.probe(table, name, precision=precision)
    P.assert_exact(p, precision, aggr='mean')
    return p


def _ref(p, name, precision, x=None):
    key = None if x is not None else ('mean', name, tuple(sorted(P.wide_options(MF, name, precision).items())))
    return _fwd_reference(p, 'mean', x=x, key=key)[0]


def _run(p, precision, x=None, **kw):
    conv = p.conv(_cls(), precision, 'mean', DEV, **kw)
    with torch.no_grad():
        out = conv((p.x[0] if x is None else x).float().to(DEV), p.ei.to(DEV), p.ea.to(DEV))
    return out, conv


def assert_equal(out, ref):
    out = out.detach().double().cpu()
    bad = (out != ref).any(1)
    assert not bool(bad.any()), ('nodes differ', torch.nonzero(bad).flatten()[:20].tolist(),
                                 float((out - ref).abs().max()))


# ---- 1. forward, every application path -------------------------------------------------------------------------------
@pytest.mark.parametrize('path', list(PATHS))
@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2'])
def test_application_paths(precision, path, lib_options, monkeypatch):
    if precision == 'f16x2' and path not in SPLIT_PATHS:
        pytest.skip('f16x2 runs the fused kernel only')
    from graph_pde_b200 import nn_conv
    opts, mods = PATHS[path]
    for k, v in opts.items():
        lib_options(k, v)
    for k, v in mods.items():
        monkeypatch.setattr(nn_conv, k, v * (2 if precision == 'f16x2' else 1))
    p = _probe(MF, 'mixed', precision)
    assert_equal(_run(p, precision)[0], _ref(p, 'mixed', precision))


def test_cuda_core_forward():
    p = _probe(MF, 'mixed', 'fp32')
    assert_equal(_run(p, 'fp32')[0], _ref(p, 'mixed', 'fp32'))


# ---- 2. graphs ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ['t2s', 'batch', 'hub_batches', 'partial_tiles'])
@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2'])
def test_graphs(precision, name, monkeypatch):
    """flow target_to_source, a block-diagonal batch, the 2,500-edge hub across ~100 flag batches, and partial last
    tiles of every box height."""
    from graph_pde_b200 import nn_conv
    if name == 'hub_batches':
        monkeypatch.setattr(nn_conv, '_Y_BYTES', 3 * 4 * 64 * 256 * 2 * (2 if precision == 'f16x2' else 1))
    p = _probe(MF, name, precision)
    assert_equal(_run(p, precision)[0], _ref(p, name, precision))


# ---- 3. formulation B, and 4. residual steps ----------------------------------------------------------------------------
def _residual(p, precision):
    """residual_step(relu_in=True) == relu(x) + mean_conv(relu(x)), bitwise."""
    xr = torch.relu(p.x[0])
    ref = _fwd_reference(p, 'mean', x=xr)[0]
    conv = p.conv(_cls(), precision, 'mean', DEV)
    with torch.no_grad():
        z = conv.residual_step(p.x[0].float().to(DEV), p.ei.to(DEV), p.ea.to(DEV), relu_in=True)
    assert_equal(z, xr + ref)


@pytest.mark.parametrize('name', ['edge_v64_src', 'edge_v64', 'edge_v32', 'edge_scalar_src', 'edge_scalar'])
@pytest.mark.parametrize('precision', ['f16', 'bf16'])
def test_formulation_b(precision, name, monkeypatch):
    """Per-edge kernel matrices: k_apply_edge_src_v / k_apply_edge_v at 64x64 and 32x32, the scalar kernels
    otherwise; plain applications and residual steps."""
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_EDGE_KERNELS', 'on')
    p = _probe(MF, name, precision)
    n0 = nn_conv.stats['edge_kernel_passes']
    assert_equal(_run(p, precision)[0], _ref(p, name, precision))
    assert nn_conv.stats['edge_kernel_passes'] > n0
    if p.cin == p.cout:
        n1 = nn_conv.stats['edge_kernel_passes']
        _residual(p, precision)
        assert nn_conv.stats['edge_kernel_passes'] > n1


@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2'])
def test_residual_step(precision):
    """residual_step (RELU_IN | RESIDUAL folded into the node prep) on formulation C."""
    _residual(_probe(MF, 'mixed', precision), precision)


# ---- 5. streamed forward ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('chunk_bytes', [3 << 20, 300007])
@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2'])
def test_streamed_edge_features(precision, chunk_bytes, monkeypatch):
    """Budget 0, half of h, and a prefix that ends inside the hub source's units."""
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_EF_WS_BYTES', chunk_bytes)
    p = _probe(MF, 'mixed', precision)
    ref = _ref(p, 'mixed', precision)
    cached, conv = _run(p, precision)
    assert_equal(cached, ref)
    hb = _h_bytes(conv, p)
    g_hub, deg_hub = hub_edges(p)
    row = hb // ((p.ei.size(1) + 127) // 128 * 128)
    straddle = (g_hub + deg_hub - 1) * row
    for budget in (0, hb // 2, straddle):
        c0 = nn_conv.stats['streamed_chunk_passes']
        out, conv = _run(p, precision, edge_feature_bytes=budget)
        assert nn_conv.stats['streamed_chunk_passes'] > c0
        if budget == straddle:
            e_res = next(iter(conv._h_cache.values())).E_res
            assert g_hub < e_res < g_hub + deg_hub, (g_hub, deg_hub, e_res)
        assert torch.equal(out, cached), budget
        assert_equal(out, ref)


# ---- 6.-8. backward -----------------------------------------------------------------------------------------------------
def _grads(name, precision):
    p = P.probe(MB, name, precision=precision)
    P.assert_exact(p, precision, aggr='mean')
    return p, _grad_reference(p, ('mean', name, precision), aggr='mean')


@pytest.mark.parametrize('name,precision', [(n, pr) for n in ('mixed', 'mixed_T1', 'mixed_T7', 'mixed_T13', 't2s', 't2s_T1',
                                                               't2s_T7', 't2s_T13')
                                            for pr in MB[n][-1] if pr != 'fp32'])
def test_tensor_core_backward(name, precision):
    """T in {1, 2, 7, 13}, both flows; x, root, bias, every W and b, and edge_attr row by row.  At f16x2, x carries
    12-bit values (non-zero lo halves)."""
    from graph_pde_b200 import nn_conv
    p, ref = _grads(name, precision)
    b0 = nn_conv.stats['mlp_backwards']
    assert_grads_equal(_library(p, precision, aggr='mean'), ref)
    assert nn_conv.stats['mlp_backwards'] > b0


@pytest.mark.parametrize('precision', ['f16', 'bf16'])
def test_batch_backward(precision):
    from graph_pde_b200 import nn_conv
    p, ref = _grads('batch', precision)
    b0 = nn_conv.stats['mlp_backwards']
    assert_grads_equal(_library(p, precision, aggr='mean'), ref)
    assert nn_conv.stats['mlp_backwards'] > b0


@pytest.mark.parametrize('name,forward', [('mixed', 'f16'), ('mixed', 'fp32'), ('t2s', 'fp32'), ('cuda_core_out32', 'f16'),
                                          ('cuda_core_out32', 'fp32'), ('cuda_core_in128', 'f16'),
                                          ('cuda_core_in128', 'fp32')])
def test_cuda_core_backward(name, forward, monkeypatch):
    """The fp32 CUDA-core backward (k_gather_g scales G by inv_deg): pinned after an f16 forward and at fp32, and
    chosen on its own for out != 64 and in > 64."""
    from graph_pde_b200 import nn_conv
    if name in ('mixed', 't2s'):
        monkeypatch.setattr(nn_conv, '_BWD_MODE', 'fp32')
    p, ref = _grads(name, forward)
    b0 = nn_conv.stats['mlp_backwards']
    assert_grads_equal(_library(p, forward, aggr='mean'), ref)
    assert nn_conv.stats['mlp_backwards'] == b0


@pytest.mark.parametrize('name', ['mixed', 't2s'])
@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2'])
def test_streamed_backward(precision, name, monkeypatch):
    """Budgets 0, half of h, and a prefix that ends inside the hub source's edges, with small chunks and batches."""
    from tests.test_gpu_exact_backward import _h_bytes as _bwd_h_bytes
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_EF_WS_BYTES', 3 << 20)
    monkeypatch.setattr(nn_conv, '_BWD_APPLY_WS_BYTES', 0)
    monkeypatch.setattr(nn_conv, '_BWD_MLP_WS_BYTES', 8 << 20)
    p, ref = _grads(name, precision)
    hb = _bwd_h_bytes(p, precision)
    g_hub, deg_hub = hub_edges(p)
    row = hb // ((p.ei.size(1) + 127) // 128 * 128)
    straddle = (g_hub + deg_hub - 1) * row
    for budget in (0, hb // 2, straddle):
        c0 = nn_conv.stats['streamed_backward_chunk_passes']
        got, conv = _library(p, precision, with_conv=True, aggr='mean', edge_feature_bytes=budget,
                             streamed_training=True)
        assert nn_conv.stats['streamed_backward_chunk_passes'] > c0, budget
        if budget == straddle:
            e_res = next(iter(conv._h_cache.values())).E_res
            assert g_hub < e_res < g_hub + deg_hub, (g_hub, deg_hub, e_res)
        assert_grads_equal(got, ref)


# ---- 9. the diagonal-kernel conv ----------------------------------------------------------------------------------------
DIAG_C, DIAG_KIN, DIAG_WIDTH = 64, 3, 64


def _diag_problem(T, flow, seed=7):
    """Small-integer diagonal-conv probe on the power-of-two graph: weights in {-1, 0, 1}, x, edge_attr and the output
    gradients small integers."""
    ei, n = P.graph('pow2_t2s' if flow == 'target_to_source' else 'pow2_mixed')
    g = torch.Generator().manual_seed(seed)
    w1 = torch.randint(-1, 2, (DIAG_WIDTH, DIAG_KIN), generator=g).double()
    b1 = torch.randint(-1, 3, (DIAG_WIDTH,), generator=g).double()
    w2 = torch.randint(-1, 2, (DIAG_C, DIAG_WIDTH), generator=g).double() * (
        torch.rand(DIAG_C, DIAG_WIDTH, generator=g) < 0.25)
    b2 = torch.randint(-2, 3, (DIAG_C,), generator=g).double()
    root = torch.randint(-1, 2, (DIAG_C, DIAG_C), generator=g).double()
    bias = torch.randint(-2, 3, (DIAG_C,), generator=g).double()
    xs = [torch.randint(-4, 5, (n, DIAG_C), generator=g).double() for _ in range(T)]
    ea = torch.randint(-2, 3, (ei.size(1), DIAG_KIN), generator=g).double()
    gouts = [torch.randint(-1, 2, (n, DIAG_C), generator=g).double() for _ in range(T)]
    return ei, n, [w1, w2], [b1, b2], root, bias, xs, ea, gouts


def _diag_budget(ei, n, ws, bs, xs, ea, gouts, flow):
    """Every node sum and parameter-gradient sum of the diagonal conv within 2^22 quanta of 2^-log2(max deg)."""
    src, dst = (ei[1], ei[0]) if flow == 'target_to_source' else (ei[0], ei[1])
    deg = torch.bincount(dst, minlength=n)
    assert bool(((deg & (deg - 1)) == 0).all())
    q = 1.0 / float(deg.max())
    inv = 1.0 / deg.clamp(min=1).double()
    hs = [ea]
    for w, b in zip(ws[:-1], bs[:-1]):
        hs.append(torch.relu(hs[-1] @ w.t() + b))
    d = hs[-1] @ ws[-1].t() + bs[-1]
    dabs = hs[-1].abs() @ ws[-1].abs().t() + bs[-1].abs()
    for x, go in zip(xs, gouts):
        node = torch.zeros(n, DIAG_C, dtype=torch.float64).index_add(0, dst, x[src].abs() * dabs * inv[dst, None])
        node += x.abs() @ torch.ones(DIAG_C, DIAG_C, dtype=torch.float64) + 2
        assert float(node.max()) / q <= P.SUM_QUANTA
        gd = (go[dst] * inv[dst, None]).abs() * x[src].abs()          # d d_e
        assert float((gd.t() @ torch.cat([hs[-1].abs(), torch.ones(len(src), 1, dtype=torch.float64)], 1)).max()) \
            / q <= P.SUM_QUANTA
        dx = torch.zeros(n, DIAG_C, dtype=torch.float64).index_add(0, src, (go[dst] * inv[dst, None]).abs() * dabs)
        assert float(dx.max()) / q <= P.SUM_QUANTA
        dz = (gd @ ws[-1].abs()) * (hs[-1] > 0)
        assert float((dz.t() @ torch.cat([hs[0].abs(), torch.ones(len(src), 1, dtype=torch.float64)], 1)).max()) \
            / q <= P.SUM_QUANTA
    assert float(d.abs().max()) < 2 ** 11


@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2', 'fp32'])
@pytest.mark.parametrize('T', [1, 2])
@pytest.mark.parametrize('flow', ['source_to_target', 'target_to_source'])
def test_diag_mean(precision, T, flow):
    """DiagNNConv mean: out, dx, root, bias, every Linear and edge_attr equal fp64 autograd through
    tests/diag_oracle.py bit for bit."""
    from graph_pde_b200.nn_conv import DiagNNConv
    from tests import diag_oracle as D
    ei, n, ws, bs, root, bias, xs, ea, gouts = _diag_problem(T, flow)
    _diag_budget(ei, n, ws, bs, xs, ea, gouts, flow)
    mlp = torch.nn.Sequential(torch.nn.Linear(DIAG_KIN, DIAG_WIDTH), torch.nn.ReLU(), torch.nn.Linear(DIAG_WIDTH, DIAG_C))
    conv = DiagNNConv(DIAG_C, DIAG_C, mlp, aggr='mean', precision=precision, flow=flow)
    with torch.no_grad():
        for lin, w, b in zip([conv.nn[0], conv.nn[2]], ws, bs):
            lin.weight.copy_(w.float())
            lin.bias.copy_(b.float())
        conv.root.copy_(root.float())
        conv.bias.copy_(bias.float())
    conv = conv.to(DEV)
    ead = ea.float().to(DEV).requires_grad_()
    eid = ei.to(DEV)
    xds = [x.float().to(DEV).requires_grad_() for x in xs]
    outs = [conv(xd, eid, ead) for xd in xds]
    sum((o * go.float().to(DEV)).sum() for o, go in zip(outs, gouts)).backward()
    wr = [w.clone().requires_grad_() for w in ws]
    br = [b.clone().requires_grad_() for b in bs]
    ear, rr, bbr = ea.clone().requires_grad_(), root.clone().requires_grad_(), bias.clone().requires_grad_()
    xrs = [x.clone().requires_grad_() for x in xs]
    refs = [D.nnconv_diag_forward(xr, ei, ear, wr, br, rr, bbr, 'mean', flow)[0] for xr in xrs]
    sum((r * go).sum() for r, go in zip(refs, gouts)).backward()
    for t in range(T):
        assert_equal(outs[t], refs[t].detach())
        assert_equal(xds[t].grad, xrs[t].grad)
    for a, b, what in [(ead.grad, ear.grad, 'edge_attr'), (conv.root.grad, rr.grad, 'root'),
                       (conv.bias.grad, bbr.grad, 'bias'), (conv.nn[0].weight.grad, wr[0].grad, 'W1'),
                       (conv.nn[0].bias.grad, br[0].grad, 'b1'), (conv.nn[2].weight.grad, wr[1].grad, 'W2'),
                       (conv.nn[2].bias.grad, br[1].grad, 'b2')]:
        assert torch.equal(a.detach().double().cpu(), b), (what, float((a.detach().double().cpu() - b).abs().max()))


# ---- 10. graph replay ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('precision', ['f16', 'f16x2'])
def test_graphed_forward_replay(precision):
    """A captured mean forward replays to the eager output and the fp64 mean bitwise."""
    from graph_pde_b200.capture import GraphedForward
    p = _probe(MF, 'mixed', precision)
    conv = p.conv(_cls(), precision, 'mean', DEV)
    x, ei, ea = p.x[0].float().to(DEV), p.ei.to(DEV), p.ea.to(DEV)
    with torch.no_grad():
        eager = conv(x, ei, ea)
    gf = GraphedForward(lambda xx: conv(xx, ei, ea), x)
    out = gf.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
    assert_equal(out, _ref(p, 'mixed', precision))
