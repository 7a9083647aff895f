"""Every backward path on exact integer probes (tests/probes.py): the probes keep every pre-activation an integer, so
the 16-bit forward computes the exact function, no ReLU mask flips, and the f16 / bf16 / f16x2 tensor-core gradients
equal fp64 autograd through the oracle bit for bit -- x, every edge-network weight and bias, root, bias, and
edge_attr row by row in the caller's edge order (a row written to the wrong edge fails)."""
import ctypes

import pytest
import torch

from oracle import nnconv_oracle as O
from tests import probes as P

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


@pytest.fixture(autouse=True)
def formulation_c(monkeypatch):
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_EDGE_KERNELS', 'off')


def _cls():
    from graph_pde_b200.nn_conv import NNConv_old
    return NNConv_old


_REF = {}


def _reference(p, key, aggr='add'):
    """fp64 autograd on the CPU of sum_t sum(conv(x_t) * g_t)."""
    if key in _REF:
        return _REF[key]
    src, dst = (t.cpu() for t in p.src_dst())
    # only edges whose target has a non-zero gradient row contribute (exact zeros elsewhere): autograd on those, with
    # the mean's in-degrees counted over every edge
    active = torch.stack([(g[dst] != 0).any(1) for g in p.grad_out]).any(0)
    inv_deg = P.in_degree_scale(p, aggr).unsqueeze(1)
    src, dst = src[active], dst[active]
    leaves = {'ea': p.ea.double().cpu()[active], 'root': p.root.clone(), 'bias': p.bias.clone()}
    for i, (w, b) in enumerate(zip(p.ws, p.bs)):
        leaves['w%d' % i], leaves['b%d' % i] = w.clone(), b.clone()
    xs = [x.clone().requires_grad_() for x in p.x]
    for v in leaves.values():
        v.requires_grad_()
    n = len(p.ws)
    loss = 0
    for x, g in zip(xs, p.grad_out):
        ws, bs = [leaves['w%d' % i] for i in range(n)], [leaves['b%d' % i] for i in range(n)]
        if aggr == 'add':
            out = O.nnconv_forward(x, torch.stack([src, dst]), leaves['ea'], ws, bs, leaves['root'], leaves['bias'],
                                   'add')
        else:                   # the active edges are every in-edge of a node with a gradient row
            out = O.nnconv_forward(x, torch.stack([src, dst]), leaves['ea'], ws, bs, None, None, 'add') * inv_deg
            out = out + x @ leaves['root'] + leaves['bias']
        loss = loss + (out * g).sum()
    loss.backward()
    ref = {k: v.grad for k, v in leaves.items()}
    ref['ea'] = torch.zeros(p.ea.shape, dtype=torch.float64).index_put_((torch.nonzero(active).flatten(),), ref['ea'])
    ref.update({'x%d' % t: x.grad for t, x in enumerate(xs)})
    _REF[key] = ref
    return ref


def _library(p, precision, with_conv=False, aggr='add', **kw):
    conv = p.conv(_cls(), precision, aggr, DEV, **kw)
    ea = p.ea.to(DEV).requires_grad_()
    ei = p.ei.to(DEV)
    xs = [x.float().to(DEV).requires_grad_() for x in p.x]
    loss = 0
    for x, g in zip(xs, p.grad_out):
        loss = loss + (conv(x, ei, ea) * g.float().to(DEV)).sum()
    loss.backward()
    lin = [m for m in conv.nn.layers if isinstance(m, torch.nn.Linear)]
    got = {'ea': ea.grad, 'root': conv.root.grad, 'bias': conv.bias.grad}
    for i, l in enumerate(lin):
        got['w%d' % i], got['b%d' % i] = l.weight.grad, l.bias.grad
    got.update({'x%d' % t: x.grad for t, x in enumerate(xs)})
    return (got, conv) if with_conv else got


def assert_grads_equal(got, ref):
    for k, r in ref.items():
        g = got[k].detach().double().cpu()
        if k == 'ea':
            bad = (g != r).any(1)
            assert not bool(bad.any()), ('edge_attr rows differ', torch.nonzero(bad).flatten()[:20].tolist())
        else:
            assert torch.equal(g, r), (k, float((g - r).abs().max()), float(r.abs().max()))


@pytest.mark.parametrize('name,precision,wide', [('mixed', 'f16', 'x'), ('mixed', 'bf16', 'x'), ('mixed', 'f16x2', 'x'),
                                                 ('mixed', 'f16x2', 'g'), ('mixed_T1', 'f16', 'x'),
                                                 ('mixed_T6', 'f16', 'x'), ('mixed_T7', 'f16', 'x'),
                                                 ('mixed_T8', 'f16', 'x'), ('mixed_T13', 'f16', 'x'),
                                                 ('asymmetric_t2s', 'f16', 'x'), ('asymmetric_t2s', 'bf16', 'x'),
                                                 ('asymmetric_t2s', 'f16x2', 'g'), ('darcy85', 'f16', 'x'),
                                                 ('darcy85', 'bf16', 'x'), ('darcy85', 'f16x2', 'x')])
def test_tensor_core_backward(name, precision, wide):
    """T in {1, 2, 6, 7, 8, 13} applications of one conv (MLP groups of 6, at most 8 applications per k_dh call), flow
    target_to_source on a graph without reverse edges, the config-2-size graph (85^2, E = 1,466,497, T = 2), and at
    f16x2 inputs (wide 'x') or output gradients (wide 'g') whose pairs have non-zero lo halves."""
    from graph_pde_b200 import nn_conv
    p = P.probe(P.BACKWARD, name, precision=precision, wide=wide)
    b0 = nn_conv.stats['mlp_backwards']
    assert_grads_equal(_library(p, precision), _reference(p, (name, precision, wide)))
    assert nn_conv.stats['mlp_backwards'] > b0                 # the tensor-core path ran


@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2'])
def test_many_backward_batches(precision, monkeypatch):
    """No per-application workspace beyond one 128-source batch, and MLP-pass batches of a few hundred edges."""
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_BWD_APPLY_WS_BYTES', 0)
    monkeypatch.setattr(nn_conv, '_BWD_MLP_WS_BYTES', 8 << 20)
    p = P.probe(P.BACKWARD, 'mixed', precision=precision)
    assert_grads_equal(_library(p, precision), _reference(p, ('mixed', precision, 'x')))


@pytest.mark.parametrize('keep', [True, False])
def test_kept_and_recomputed_hidden_activations(keep, monkeypatch):
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_KEEP_ACTS_MAX_BYTES', (8 << 30) if keep else 0)
    p = P.probe(P.BACKWARD, 'mixed')
    assert_grads_equal(_library(p, 'f16'), _reference(p, ('mixed', 'f16', 'x')))


def _h_bytes(p, precision):
    from graph_pde_b200 import _lib, nn_conv
    conv = p.conv(_cls(), precision, 'add', DEV)
    plan = nn_conv.get_plan(p.ei.to(DEV), p.n_nodes, conv.flow)
    prep = conv._get_prepared(precision)
    h_b, ws_b = ctypes.c_size_t(), ctypes.c_size_t()
    _lib.check(_lib.lib().nnconv_edge_features_sizes(plan.handle, prep.handle, 1 << 20, ctypes.byref(h_b),
                                                     ctypes.byref(ws_b)))
    return h_b.value


@pytest.mark.parametrize('name', ['mixed', 'asymmetric_t2s'])
@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2'])
def test_streamed_backward(precision, name, monkeypatch):
    """Budgets 0, half of h, and a prefix that ends inside the hub source's edges (the straddling source is recomputed
    whole), with small chunks and batches.  Under target_to_source the hub source is the graph's hub target."""
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_EF_WS_BYTES', 3 << 20)
    monkeypatch.setattr(nn_conv, '_BWD_APPLY_WS_BYTES', 0)
    monkeypatch.setattr(nn_conv, '_BWD_MLP_WS_BYTES', 8 << 20)
    wide = 'g' if name == 'asymmetric_t2s' else 'x'
    p = P.probe(P.BACKWARD, name, precision=precision, wide=wide)
    ref = _reference(p, (name, precision, wide))
    hb = _h_bytes(p, precision)
    g_hub, deg_hub = hub_edges(p)
    row = hb // ((p.ei.size(1) + 127) // 128 * 128)          # h bytes per edge row
    straddle = (g_hub + deg_hub - 1) * row                    # E_res: a unit boundary inside the hub
    for budget in (0, hb // 2, straddle):
        c0 = nn_conv.stats['streamed_backward_chunk_passes']
        got, conv = _library(p, precision, with_conv=True, edge_feature_bytes=budget, streamed_training=True)
        assert nn_conv.stats['streamed_backward_chunk_passes'] > c0, budget
        if budget == straddle:
            e_res = next(iter(conv._h_cache.values())).E_res
            assert g_hub < e_res < g_hub + deg_hub, (g_hub, deg_hub, e_res)
        assert_grads_equal(got, ref)


def hub_edges(p):
    """(sorted edges before the largest source, its out-degree) in the library's source order."""
    src, _ = p.src_dst()
    counts = torch.bincount(src.cpu(), minlength=p.n_nodes)
    hub = int(counts.argmax())
    return int(counts[:hub].sum()), int(counts[hub])


@pytest.mark.parametrize('name,precision', [('mixed', 'f16'), ('mixed', 'fp32'), ('cuda_core_out32', 'f16'),
                                            ('cuda_core_in128', 'f16'), ('cuda_core_in128', 'fp32')])
def test_cuda_core_backward(name, precision, monkeypatch):
    """The fp32 CUDA-core backward: pinned by NNCONV_B200_BACKWARD=fp32, and chosen for out != 64 and in > 64."""
    from graph_pde_b200 import nn_conv
    if name == 'mixed':
        monkeypatch.setattr(nn_conv, '_BWD_MODE', 'fp32')
    p = P.probe(P.BACKWARD, name)
    b0 = nn_conv.stats['mlp_backwards']
    assert_grads_equal(_library(p, precision), _reference(p, name))
    assert nn_conv.stats['mlp_backwards'] == b0                # no tensor-core MLP pass
