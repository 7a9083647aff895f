"""aggr='max' on the GPU.  On the exact probes of tests/probes.py (exact for max, see tests/test_aggr_max_host.py) the
library's out and argmax must equal the fp64 reference of tests/max_oracle.py bit for bit on every application path,
and every gradient must equal fp64 autograd through that reference.  Integer messages tie often, so the tie rule is
exercised, not avoided.  On random data the forward is within the add tolerance (max is 1-Lipschitz in the messages)
and the gradients within the existing bounds, against the reference's backward given the library's argmax."""
import pytest
import torch

from tests import max_oracle as M
from tests import probes as P
from tests.helpers import TOL

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


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


def _cls():
    from graph_pde_b200.nn_conv import NNConv_old
    return NNConv_old


def _reference(p, x=None):
    src, dst = (t.cpu() for t in p.src_dst())
    x = p.x[0] if x is None else x
    return M.nnconv_forward_max(x, torch.stack([src, dst]), p.ea.double().cpu(), p.ws, p.bs, p.root, p.bias)


def _run(p, precision, x=None, flags=0, **kw):
    conv = p.conv(_cls(), precision, 'max', DEV, **kw)
    x = p.x[0] if x is None else x
    with torch.no_grad():
        out, am = conv._forward_impl(x.float().to(DEV), p.ei.to(DEV), p.ea.to(DEV), flags=flags, with_argmax=True)
    return out, am, conv


def _assert_exact(out, am, ref, ref_am):
    out, am = out.double().cpu(), am.cpu().to(torch.int64)
    bad = (out != ref).any(1) | (am != ref_am).any(1)
    assert not bool(bad.any()), ('nodes differ', torch.nonzero(bad).flatten()[:20].tolist())


def _custom(cin, cout=64, precision='f16'):
    ei, n = P.graph('mixed')
    return P.make_probe(ei, n, [6, 64, 128, cin * cout], cin, cout)


# ---- forward on exact probes -------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name,precision', [('mixed', pr) for pr in ('f16', 'bf16', 'f16x2', 'fp32')] +
                         [(n, pr) for n in ('partial_tiles', 'asymmetric_t2s', 'batch', 'nc16', 'nc32', 'nc48')
                          for pr in ('f16', 'bf16', 'f16x2')] +
                         [('out128', 'f16'), ('out128', 'bf16'), ('kp1088', 'f16'), ('kp1088', 'bf16')])
def test_forward_exact(name, precision):
    """The fused kernel at out 16 / 32 / 48 / 64, k_conv_tc at out 128 and Kp 1088, the fp32 CUDA-core path; partial
    tiles of every box height, ten copies of one edge (exact ties), target_to_source and a block-diagonal batch."""
    p = P.probe(P.FORWARD, name, precision=precision)
    ref, ref_am = _reference(p)
    assert M.win_share(ref_am, p.ei.size(1)) >= 0.5
    out, am, _ = _run(p, precision)
    _assert_exact(out, am, ref, ref_am)


@pytest.mark.parametrize('cin', [1, 128])
@pytest.mark.parametrize('precision', ['f16', 'f16x2'])
def test_forward_exact_in_channels(cin, precision):
    p = _custom(cin)
    P.assert_exact(p, precision)
    ref, ref_am = _reference(p)
    out, am, _ = _run(p, precision)
    _assert_exact(out, am, ref, ref_am)


@pytest.mark.parametrize('precision', ['f16', 'bf16'])
def test_fused_equals_per_batch(precision, lib_options):
    p = P.probe(P.FORWARD, 'mixed', precision=precision)
    fused, am_f, _ = _run(p, precision)
    lib_options('no_fuse', 1)
    chain, am_c, _ = _run(p, precision)
    assert torch.equal(fused, chain) and torch.equal(am_f, am_c)


@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2'])
def test_streamed_equals_cached(precision, monkeypatch):
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_EF_WS_BYTES', 3 << 20)
    p = P.probe(P.FORWARD, 'mixed', precision=precision)
    cached, am, conv = _run(p, precision)
    h_b = next(iter(conv._h_cache.values())).h.numel()
    for budget in (0, h_b // 2):
        c0 = nn_conv.stats['streamed_chunk_passes']
        out, am_s, _ = _run(p, precision, edge_feature_bytes=budget)
        assert nn_conv.stats['streamed_chunk_passes'] > c0
        assert torch.equal(out, cached) and torch.equal(am_s, am), budget
    ref, ref_am = _reference(p)
    _assert_exact(cached, am, ref, ref_am)


@pytest.mark.parametrize('precision', ['f16', 'f16x2'])
def test_residual_step_and_graph_replay(precision):
    from graph_pde_b200.capture import GraphedForward
    p = P.probe(P.FORWARD, 'mixed')
    xr = torch.relu(p.x[0])
    ref, _ = _reference(p, x=xr)
    conv = p.conv(_cls(), precision, 'max', DEV)
    x, ei, ea = p.x[0].float().to(DEV), p.ei.to(DEV), p.ea.to(DEV)
    with torch.no_grad():
        z = conv.residual_step(x, ei, ea, relu_in=True)
        eager = conv(x, ei, ea)
    assert torch.equal(z.double().cpu(), xr + ref)
    gf = GraphedForward(lambda xx: conv(xx, ei, ea), x)
    out = gf.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)


def test_low_degree_graph_runs_formulation_c():
    from graph_pde_b200 import nn_conv
    p = P.probe(P.FORWARD, 'edge_v64')
    n0 = nn_conv.stats['edge_kernel_passes']
    out, am, _ = _run(p, 'f16')
    assert nn_conv.stats['edge_kernel_passes'] == n0
    ref, ref_am = _reference(p)
    _assert_exact(out, am, ref, ref_am)


# ---- gradients on exact probes -----------------------------------------------------------------------------------------
def _grad_reference(p, argmaxes=None):
    """fp64 autograd through the reference over the probe's T applications (each with its own x and grad_out)."""
    src, dst = p.src_dst()
    ei = torch.stack([src.cpu(), dst.cpu()])
    ws = [w.clone().requires_grad_(True) for w in p.ws]
    bs = [b.clone().requires_grad_(True) for b in p.bs]
    root = p.root.clone().requires_grad_(True)
    bias = p.bias.clone().requires_grad_(True)
    ea = p.ea.double().cpu().requires_grad_(True)
    xs = [x.clone().requires_grad_(True) for x in p.x]
    loss = 0
    for t in range(p.T):
        out, _ = M.nnconv_forward_max(xs[t], ei, ea, ws, bs, root, bias,
                                      argmax=None if argmaxes is None else argmaxes[t])
        loss = loss + (out * p.grad_out[t]).sum()
    loss.backward()
    return {'x': [x.grad for x in xs], 'ws': [w.grad for w in ws], 'bs': [b.grad for b in bs], 'root': root.grad,
            'bias': bias.grad, 'ea': ea.grad}


def _grad_library(p, precision, **kw):
    conv = p.conv(_cls(), precision, 'max', DEV, **kw)
    ea = p.ea.to(DEV).requires_grad_(True)
    xs = [x.float().to(DEV).requires_grad_(True) for x in p.x]
    ei = p.ei.to(DEV)
    loss = 0
    for t in range(p.T):
        loss = loss + (conv(xs[t], ei, ea) * p.grad_out[t].float().to(DEV)).sum()
    loss.backward()
    lins = [m for m in conv.nn.modules() if isinstance(m, torch.nn.Linear)]
    return {'x': [x.grad for x in xs], 'ws': [l.weight.grad for l in lins], 'bs': [l.bias.grad for l in lins],
            'root': conv.root.grad, 'bias': conv.bias.grad, 'ea': ea.grad}


def _flat(g):
    out = []
    for k in ('x', 'ws', 'bs', 'root', 'bias', 'ea'):
        v = g[k]
        for i, t in enumerate(v if isinstance(v, list) else [v]):
            out.append(('%s%d' % (k, i), t.double().cpu()))
    return out


@pytest.mark.parametrize('name,precision,mode', [('mixed', 'f16', 'tc'), ('mixed', 'bf16', 'tc'), ('mixed', 'f16x2', 'tc'),
                                                 ('asymmetric_t2s', 'f16', 'tc'), ('cuda_core_out32', 'fp32', 'fp32'),
                                                 ('cuda_core_out32', 'f16', 'fp32'), ('cuda_core_in128', 'fp32', 'fp32')])
def test_gradients_exact(name, precision, mode, monkeypatch):
    """T = 2 applications of one conv (one MLP pass routes by two different argmaxes), edge_attr included: bitwise
    against fp64 autograd through the reference."""
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_BWD_MODE', mode)
    p = P.probe(P.BACKWARD, name, precision=precision)
    ref = _grad_reference(p)
    got = _grad_library(p, precision)
    for (k, a), (_, b) in zip(_flat(got), _flat(ref)):
        assert torch.equal(a, b), (k, float((a - b).abs().max()))


@pytest.mark.parametrize('precision', ['f16', 'f16x2'])
def test_streamed_training_gradients_exact(precision, monkeypatch):
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_EF_WS_BYTES', 3 << 20)
    p = P.probe(P.BACKWARD, 'mixed', precision=precision)
    ref = _grad_reference(p)
    conv = p.conv(_cls(), precision, 'max', DEV)
    with torch.no_grad():
        conv(p.x[0].float().to(DEV), p.ei.to(DEV), p.ea.to(DEV))
    h_b = next(iter(conv._h_cache.values())).h.numel()
    for budget in (0, h_b // 2):
        c0 = nn_conv.stats['streamed_backward_chunk_passes']
        got = _grad_library(p, precision, edge_feature_bytes=budget, streamed_training=True)
        assert nn_conv.stats['streamed_backward_chunk_passes'] > c0
        for (k, a), (_, b) in zip(_flat(got), _flat(ref)):
            assert torch.equal(a, b), (budget, k, float((a - b).abs().max()))


# ---- random data -------------------------------------------------------------------------------------------------------
def _random_probe(seed, cin=64, cout=64):
    g = torch.Generator().manual_seed(seed)
    ei, n = P.graph('mixed')
    p = P.make_probe(ei, n, [6, 64, 128, cin * cout], cin, cout, T=1, grad=True)
    p.ea = torch.rand(ei.size(1), 6, generator=g) * 2 - 1
    p.ws = [torch.randn(w.shape, generator=g, dtype=torch.float64) / w.shape[1] ** 0.5 for w in p.ws]
    p.bs = [torch.randn(b.shape, generator=g, dtype=torch.float64) * 0.1 for b in p.bs]
    p.x = [torch.randn(n, cin, generator=g, dtype=torch.float64)]
    p.grad_out = [torch.randn(n, cout, generator=g, dtype=torch.float64)]
    return p


@pytest.mark.parametrize('precision,mode', [('f16', 'tc'), ('bf16', 'tc'), ('f16x2', 'tc'), ('fp32', 'fp32')])
def test_random_data(precision, mode, monkeypatch):
    """Forward within TOL[precision] of the reference; an argmax that differs from the reference's is a near-tie (the
    two reference messages within the forward tolerance); gradients within the add tolerances against the
    reference's backward routed by the library's argmax."""
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_BWD_MODE', mode)
    p = _random_probe(11)
    out, am, _ = _run(p, precision)
    ref, ref_am = _reference(p)
    scale = float(ref.abs().max())
    tol = TOL[precision]
    assert float((out.double().cpu() - ref).abs().max()) <= tol * scale
    am = am.cpu().to(torch.int64)
    diff = am != ref_am
    src, dst = p.src_dst()
    msg = M.messages(p.x[0], src.cpu(), p.ea.double(), p.ws, p.bs, p.cin, p.cout)
    col = torch.arange(p.cout).expand_as(am)
    gap = (msg[am[diff], col[diff]] - msg[ref_am[diff], col[diff]]).abs()
    assert float(gap.max()) <= tol * scale if gap.numel() else True
    assert float(diff.double().mean()) < 0.05
    ref_g = _grad_reference(p, argmaxes=[am])
    got = _grad_library(p, precision)
    # the bounds of the add / mean backward tests against the exact fp64 oracle: the tensor cores at 16 bits
    # (test_gpu_backward_tc.GTOL_EXACT), f16x2, and the CUDA-core backward (test_gpu_backward)
    bound = {'f16': 8e-2, 'bf16': 8e-2, 'f16x2': 1e-4, 'fp32': 5e-4}[precision]
    for (k, a), (_, b) in zip(_flat(got), _flat(ref_g)):
        err = float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30)
        print('random %s %s: max|g - ref| / max|ref| = %.3e' % (precision, k, err))
        if k == 'ea0' and precision in ('f16', 'bf16'):
            # test_gpu_edge_attr_grad's bounds for the edge_attr gradient at 16 bits against the exact oracle (a
            # per-edge gradient: one rounded dz_1 row moves its entry, so max-relative 0.3 and L2-relative 5e-2)
            l2 = float((a - b).norm() / b.norm())
            assert err < 0.3 and l2 < 5e-2, (k, err, l2)
        else:
            assert err <= bound, (k, err)


# ---- a captured training step ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('precision,width', [('f16x2', 64), ('fp32', 32)])
def test_graphed_train_step_matches_eager(precision, width):
    """A KernelNN with aggr='max' (width 64: tensor-core backward; 32: CUDA-core), replayed from a CUDA graph against
    eager steps, within the bounds of the add / mean replay tests: the loss of every step and the first step's
    gradients.  Under max most entries of dW_L are exact zeros plus fp32 atomic-order noise, and Adam's first steps
    move such an entry by about lr whatever its size; as at f16 in test_gpu_graphed_train, the parameters after the
    steps are not compared."""
    import torch.nn.functional as F
    from graph_pde_b200 import GraphedTrainStep
    from graph_pde_b200.models import KernelNN
    from tests.helpers import rel_err

    class _Data(object):
        pass

    def model():
        torch.manual_seed(0)
        m = KernelNN(width, 64, 3, 6, in_width=6, precision=precision).to(DEV)
        m.conv1.aggr = 'max'
        return m

    model_e, model_g = model(), model()
    model_g.load_state_dict(model_e.state_dict())
    opt_e = torch.optim.Adam(model_e.parameters(), lr=1e-3, capturable=True)
    opt_g = torch.optim.Adam(model_g.parameters(), lr=1e-3, capturable=True)
    ei, n = P.graph('mixed')
    gen = torch.Generator().manual_seed(3)
    d = _Data()
    d.x, d.edge_index, d.edge_attr = torch.rand(n, 6, generator=gen).to(DEV), ei.to(DEV), \
        torch.rand(ei.size(1), 6, generator=gen).to(DEV)
    y = torch.randn(n, 1, generator=gen).to(DEV)
    dg = _Data()
    dg.x, dg.edge_index, dg.edge_attr = d.x.clone(), d.edge_index.clone(), d.edge_attr.clone()
    yg = y.clone()

    def loss_of(m):
        return lambda dd, yy: F.mse_loss(m(dd).view(-1), yy.view(-1))

    step = GraphedTrainStep(loss_of(model_g), model_g, opt_g, dg, yg)
    for i in range(4):
        opt_e.zero_grad(set_to_none=True)
        loss_e = loss_of(model_e)(d, y)
        loss_e.backward()
        opt_e.step()
        loss_g = step.replay()
        assert rel_err(loss_g, loss_e.detach()) < TOL[precision], (i, float(loss_g), float(loss_e))
        if i == 0:
            for (name, pg), pe in zip(model_g.named_parameters(), model_e.parameters()):
                assert rel_err(pg.grad, pe.grad) < TOL[precision], (name, rel_err(pg.grad, pe.grad))


# ---- full scale --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('budget', [None, 24 << 30])
def test_darcy241_one_application(budget):
    """One f16 application at 241^2 (24.6 M edges, ~423 in-edges per node: at most 64 of a node's edges can win, so
    the share of winning edges is bounded by 64 / 423 here), whole h and a 24 GB budget, bitwise in out and argmax
    against the reference computed edge-chunked on the GPU."""
    import gc
    from graph_pde_b200 import nn_conv
    nn_conv.clear_caches()
    gc.collect()
    p = P.probe(P.FORWARD, 'darcy241', DEV)
    kw = {} if budget is None else {'edge_feature_bytes': budget}
    c0 = nn_conv.stats['streamed_chunk_passes']
    out, am, conv = _run(p, 'f16', **kw)
    assert (nn_conv.stats['streamed_chunk_passes'] > c0) == (budget is not None)
    out, am = out.cpu(), am.cpu().to(torch.int64)
    conv.invalidate()
    del conv
    torch.cuda.empty_cache()
    x = p.x[0].to(DEV)
    src, dst = p.src_dst()
    ws, bs = [w.to(DEV) for w in p.ws], [b.to(DEV) for b in p.bs]
    n, cout, e = p.n_nodes, p.cout, src.numel()
    best = torch.full((n, cout), float('-inf'), dtype=torch.float64, device=DEV)
    arg = torch.full((n, cout), -1, dtype=torch.int64, device=DEV)
    step = 1 << 16
    for s in range(0, e, step):            # chunks in caller order: a strict > keeps the earlier index on a tie
        msg = M.messages(x, src[s:s + step], p.ea[s:s + step].double(), ws, bs, p.cin, cout)
        am_c = M.winners(msg, dst[s:s + step], n)
        has = am_c >= 0
        val = msg.gather(0, am_c.clamp(min=0))
        take = has & (val > best)
        best = torch.where(take, val, best)
        arg = torch.where(take, am_c + s, arg)
    ref = torch.where(arg >= 0, best, torch.zeros_like(best)) + x @ p.root.to(DEV) + p.bias.to(DEV)
    ref, arg = ref.cpu(), arg.cpu()
    bad = (out.double() != ref).any(1) | (am != arg).any(1)
    assert not bool(bad.any()), ('nodes differ', int(bad.sum()), torch.nonzero(bad).flatten()[:20].tolist())
