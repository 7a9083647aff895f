"""Training on streamed edge features (streamed_training=True): the tensor-core backward over a partially resident h
(nnconv_backward_apply_streamed / nnconv_backward_mlp_streamed) recomputes the h of the streamed edges per source batch
with the forward's GEMMs, so its gradients are those of the cached backward up to the order of fp32 atomics.  Small
budgets, small chunks and small backward workspaces make small graphs stream over many batches."""
import ctypes

import pytest
import torch

from tests.helpers import DenseNetLike, make_conv
from tests.test_gpu_backward_f16x2 import (CFG2_GTOL, CFG2_GTOL_EA, CFG2_GTOL_EA_L2, _check, _Data, _kernelnn_step,
                                           _oracle_grads, _problem, _relerr, _relerr_l2, _run)

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
GRAD_TOL = 1e-5        # streamed vs cached backward on identical inputs: fp32 atomic order only
STEP_TOL = 1e-4        # a whole f16x2 KernelNN step: the forward chains differ in fp32 atomic order
F16_STEP_TOL = 3e-3    # the same at f16: such a difference can round to a neighbouring 16-bit operand


@pytest.fixture
def small(monkeypatch):
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_EDGE_KERNELS', 'off')
    monkeypatch.setattr(nn_conv, '_EF_WS_BYTES', 3 << 20)       # chunks of a few thousand edges
    monkeypatch.setattr(nn_conv, '_BWD_APPLY_WS_BYTES', 0)      # 128-source batches in the per-application backward
    monkeypatch.setattr(nn_conv, '_BWD_MLP_WS_BYTES', 8 << 20)  # several batches in the MLP pass


def _cls():
    from graph_pde_b200.nn_conv import NNConv_old
    return NNConv_old


def _conv(precision, aggr, rb, layers=(6, 128, 128, 64 * 64), w=64, seed=11):
    torch.manual_seed(seed)
    lin = [m for m in DenseNetLike(list(layers)).layers if isinstance(m, torch.nn.Linear)]
    ws, bs = [l.weight.detach().clone() for l in lin], [l.bias.detach().clone() for l in lin]
    root = torch.randn(w, layers[-1] // w) * 0.1 if rb else None
    bias = torch.randn(layers[-1] // w) * 0.1 if rb else None
    return make_conv(_cls(), ws, bs, root, bias, aggr, w, layers[-1] // w, precision, DEV)


def _ball(s, r, seed=0):
    from graph_pde_b200 import graphs
    ei = graphs.ball_connectivity(s, r, DEV, True)
    _, _, ea = graphs.darcy_sample(s, r, DEV, seed=seed, edge_index=ei)
    return ei, ea


def _hub_graph(N=300, E=5000, k_in=6, seed=5):
    """Unsorted edges, a hub source (7) with 1500 out-edges, duplicates, isolated nodes."""
    gen = torch.Generator().manual_seed(seed)
    src = torch.randint(0, N - 20, (E,), generator=gen)
    dst = torch.randint(10, N, (E,), generator=gen)
    src[:1500] = 7
    return torch.stack([src, dst]).to(DEV), torch.randn(E, k_in, generator=gen).to(DEV)


def _plan_prep(conv, ei, n):
    from graph_pde_b200 import nn_conv
    return nn_conv.get_plan(ei, n, conv.flow), conv._get_prepared(conv.precision)


def _h_bytes(conv, ei, n):
    from graph_pde_b200 import _lib
    plan, prep = _plan_prep(conv, ei, n)
    h_b, ws_b = ctypes.c_size_t(), ctypes.c_size_t()
    _lib.check(_lib.lib().nnconv_edge_features_sizes(plan.handle, prep.handle, 1 << 20, ctypes.byref(h_b),
                                                     ctypes.byref(ws_b)))
    return h_b.value


def _grads(conv, ei, ea, xs, wts, budget, streamed=True):
    """Gradients of sum_k <conv(x_k), w_k> (one shared conv, fixed leaf inputs) with the given cache budget, and the
    forward / backward chunk passes it took."""
    from graph_pde_b200 import nn_conv
    conv.edge_feature_bytes = budget
    conv.streamed_training = streamed
    conv.invalidate()
    conv._tstate = None
    conv.zero_grad(set_to_none=True)
    f0, b0 = nn_conv.stats['streamed_chunk_passes'], nn_conv.stats['streamed_backward_chunk_passes']
    ead = ea.clone().requires_grad_(True)
    xl = [x.clone().requires_grad_(True) for x in xs]
    sum((conv(x, ei, ead) * w).sum() for x, w in zip(xl, wts)).backward()
    g = {'x%d' % k: x.grad for k, x in enumerate(xl)}
    g['edge_attr'] = ead.grad
    g.update({k: p.grad for k, p in conv.named_parameters()})
    return g, nn_conv.stats['streamed_chunk_passes'] - f0, nn_conv.stats['streamed_backward_chunk_passes'] - b0


def _assert_close(got, ref, tol=GRAD_TOL):
    errs = {k: _relerr(got[k], ref[k]) for k in ref}
    assert all(v <= tol for v in errs.values()), errs


def _inputs(n, w, T, aggr, seed=2):
    gen = torch.Generator().manual_seed(seed)
    xs = [torch.randn(n, w, generator=gen).to(DEV) * (0.05 if aggr == 'add' else 1.0) for _ in range(T)]
    wts = [torch.randn(n, 64, generator=gen).to(DEV) for _ in range(T)]
    return xs, wts


@pytest.mark.parametrize('flow', ['source_to_target', 'target_to_source'])
@pytest.mark.parametrize('root_bias', [True, False])
@pytest.mark.parametrize('aggr', ['mean', 'add'])
@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2'])
def test_isolated_applications_streamed_vs_cached(small, precision, aggr, root_bias, flow):
    """T = 3 applications of one conv to fixed inputs: gradients of every x_k, every parameter and edge_attr with
    budgets 0 and half of h against the cached run."""
    ei, ea = _ball(20, 0.25)
    conv = _conv(precision, aggr, root_bias)
    conv.flow = flow
    xs, wts = _inputs(400, 64, 3, aggr)
    ref, nf, nb = _grads(conv, ei, ea, xs, wts, None)
    assert nf == 0 and nb == 0
    hb = _h_bytes(conv, ei, 400)
    for budget in (0, hb // 2):
        got, nf, nb = _grads(conv, ei, ea, xs, wts, budget)
        assert nf >= 3 and nb >= 3 + 1, (budget, nf, nb)
        _assert_close(got, ref)


@pytest.mark.parametrize('precision', ['f16', 'f16x2'])
def test_hub_source_straddles_prefix(small, precision):
    """A source with more out-edges (1500) than one chunk of the request holds, with E_res inside its edges: the
    sizes query grows the chunk to the largest source and the straddling source is recomputed whole."""
    from graph_pde_b200 import _lib, nn_conv
    L = _lib.lib()
    ei, ea = _hub_graph()
    conv = _conv(precision, 'mean', True, layers=(6, 128, 64, 64 * 64))
    xs, wts = _inputs(300, 64, 2, 'mean', seed=4)
    ref, _, _ = _grads(conv, ei, ea, xs, wts, None)
    plan, prep = _plan_prep(conv, ei, 300)
    assert plan.max_out_deg >= 1500
    hrow = 64 * 2 * (2 if precision == 'f16x2' else 1)
    cached, streamed = ctypes.c_size_t(), ctypes.c_size_t()
    _lib.check(L.nnconv_backward_apply_sizes(plan.handle, prep.handle, 0, ctypes.byref(cached)))
    _lib.check(L.nnconv_backward_apply_streamed_sizes(plan.handle, prep.handle, 0, 0, 0, ctypes.byref(streamed)))
    assert streamed.value - cached.value >= (plan.max_out_deg + 127) // 128 * 128 * hrow
    g_hub = int((ei[0] < 7).sum())                       # sorted edges of the sources before the hub
    got, nf, nb = _grads(conv, ei, ea, xs, wts, (g_hub + 700) * hrow)
    st = next(v[0] for v in conv._h_cache.values())
    assert isinstance(st, nn_conv._Streamed) and g_hub < st.E_res < g_hub + 1500, (g_hub, st.E_res)
    assert nf >= 2 and nb >= 3
    _assert_close(got, ref)


def test_f16x2_streamed_vs_oracle(small):
    """f16x2, every edge streamed, against the exact fp64 oracle within the tensor-core backward's own bound."""
    ei, ea, x, ws, bsl, root, bias, _ = _problem([6, 128, 128, 32 * 64], 32, True, True)
    gen = torch.Generator().manual_seed(9)
    xs = [x] + [torch.randn(x.shape, generator=gen) for _ in range(2)]
    gouts = [torch.randn(x.size(0), 64, generator=gen) for _ in range(3)]
    ref = _oracle_grads(ei, ea, xs, gouts, ws, bsl, root, bias, 'mean')
    conv = make_conv(_cls(), ws, bsl, root, bias, 'mean', 32, 64, 'f16x2', DEV)
    conv.edge_feature_bytes = 0
    conv.streamed_training = True
    from graph_pde_b200 import nn_conv
    b0 = nn_conv.stats['streamed_backward_chunk_passes']
    got = _run(conv, ei, ea, xs, gouts)
    assert nn_conv.stats['streamed_backward_chunk_passes'] > b0
    _check(got, ref)


def test_oom_fallback_streams_in_training_only_with_option(small, monkeypatch):
    """The whole h "does not fit" (simulated OOM): without the option training raises as before, with it the step
    streams and matches the cached gradients."""
    ei, ea = _ball(20, 0.25)
    conv = _conv('f16', 'mean', True)
    xs, wts = _inputs(400, 64, 2, 'mean')
    ref, _, _ = _grads(conv, ei, ea, xs, wts, None)
    hb = _h_bytes(conv, ei, 400)
    real_empty = torch.empty

    def empty_oom(*args, **kw):
        if args and args[0] == hb:
            raise torch.cuda.OutOfMemoryError('simulated: h does not fit')
        return real_empty(*args, **kw)
    monkeypatch.setattr(torch, 'empty', empty_oom)
    with pytest.raises(RuntimeError, match='training needs the whole h resident'):
        _grads(conv, ei, ea, xs, wts, None, streamed=False)
    got, nf, nb = _grads(conv, ei, ea, xs, wts, None)
    monkeypatch.setattr(torch, 'empty', real_empty)
    assert nf >= 2 and nb >= 3
    _assert_close(got, ref)


@pytest.mark.parametrize('case', ['bwd_fp32', 'out32'])
def test_cuda_core_backward_under_streamed_forward(small, monkeypatch, case):
    """The CUDA-core backward (NNCONV_B200_BACKWARD=fp32, or a conv the tensor-core backward does not cover) recomputes
    everything from edge_attr: under a streamed forward it matches its cached run."""
    from graph_pde_b200 import nn_conv
    if case == 'bwd_fp32':
        monkeypatch.setattr(nn_conv, '_BWD_MODE', 'fp32')
        conv = _conv('f16', 'mean', True)
    else:
        conv = _conv('f16', 'mean', True, layers=(6, 128, 128, 64 * 32))
        assert not conv._get_prepared('f16').bwd_tc
    ei, ea = _ball(20, 0.25)
    xs, wts = _inputs(400, 64, 2, 'mean')
    wts = [w_[:, :conv.out_channels].contiguous() for w_ in wts]
    ref, _, _ = _grads(conv, ei, ea, xs, wts, None)
    got, nf, nb = _grads(conv, ei, ea, xs, wts, _h_bytes(conv, ei, 400) // 2)
    assert nf >= 2 and nb == 0
    _assert_close(got, ref)


def _kernelnn(s, r, precision, seed=2):
    from graph_pde_b200 import graphs
    from graph_pde_b200.models import KernelNN
    ei = graphs.ball_connectivity(s, r, DEV, True)
    node_x, _, ea = graphs.darcy_sample(s, r, DEV, seed=seed, edge_index=ei)
    torch.manual_seed(0)
    model = KernelNN(64, 1024, 6, 6, in_width=node_x.size(1), precision=precision).to(DEV)
    y = torch.randn(s * s, 1, generator=torch.Generator().manual_seed(1)).to(DEV)
    d = _Data()
    d.x, d.edge_index, d.edge_attr = node_x, ei, ea
    return model, d, y


def _step(model, d, y, budget, monkeypatch, mode='auto', streamed=True):
    from graph_pde_b200 import nn_conv
    model.conv1.edge_feature_bytes = budget
    model.conv1.streamed_training = streamed
    f0, b0 = nn_conv.stats['streamed_chunk_passes'], nn_conv.stats['streamed_backward_chunk_passes']
    g = _kernelnn_step(model, d, y, mode, monkeypatch)
    passes = (nn_conv.stats['streamed_chunk_passes'] - f0, nn_conv.stats['streamed_backward_chunk_passes'] - b0)
    model.conv1.invalidate()
    torch.cuda.empty_cache()
    return g, passes


def test_darcy85_f16x2_kernelnn_step_streamed(monkeypatch):
    """KernelNN(w=64, ker_width=1024, T=6) on the 85x85, r=0.10 graph at f16x2 with half of h resident against the
    cached step: every parameter in the max norm, edge_attr in the 2-norm."""
    model, d, y = _kernelnn(85, 0.10, 'f16x2')
    ref, passes = _step(model, d, y, None, monkeypatch)
    assert passes == (0, 0)
    hb = _h_bytes(model.conv1, d.edge_index, 85 * 85)
    got, passes = _step(model, d, y, hb // 2, monkeypatch)
    assert passes[0] >= 6 and passes[1] >= 7, passes
    errs = {k: _relerr(got[k], ref[k]) for k in ref if k != 'edge_attr'}
    errs['edge_attr(l2)'] = _relerr_l2(got['edge_attr'], ref['edge_attr'])
    assert all(v <= STEP_TOL for v in errs.values()), errs


def test_darcy241_f16_kernelnn_step_streamed(monkeypatch):
    """241x241, r=0.05 (E = 24,557,297) at f16 with a 24 GB prefix against the cached step (h is 47 GiB and fits)."""
    model, d, y = _kernelnn(241, 0.05, 'f16', seed=3)
    ref, passes = _step(model, d, y, None, monkeypatch)
    assert passes == (0, 0)
    got, passes = _step(model, d, y, 24 * 10 ** 9, monkeypatch)
    assert passes[0] >= 6 and passes[1] >= 7, passes
    errs = {k: _relerr(got[k], ref[k]) for k in ref if k != 'edge_attr'}
    assert all(v <= F16_STEP_TOL for v in errs.values()), errs


def test_darcy241_f16x2_kernelnn_step_auto_budget(monkeypatch):
    """The fp32-grade training step at the headline size: f16x2 edge features of 241x241 are 94 GiB, so the automatic
    policy streams (no OOM in the forward or in loss.backward()).  Gradients against the CUDA-core backward of the same
    streamed forward, within the config-2 bounds."""
    model, d, y = _kernelnn(241, 0.05, 'f16x2', seed=3)
    got, passes = _step(model, d, y, None, monkeypatch)
    assert passes[0] >= 6 and passes[1] >= 7, passes
    assert all(bool(torch.isfinite(v).all()) for v in got.values())
    ref, passes = _step(model, d, y, None, monkeypatch, mode='fp32')
    assert passes[0] >= 6 and passes[1] == 0, passes
    errs = {k: _relerr(got[k], ref[k]) for k in ref}
    bad = {k: v for k, v in errs.items() if not v < (CFG2_GTOL_EA if k == 'edge_attr' else CFG2_GTOL)}
    l2 = _relerr_l2(got['edge_attr'], ref['edge_attr'])
    assert not bad and l2 < CFG2_GTOL_EA_L2, (errs, l2)
