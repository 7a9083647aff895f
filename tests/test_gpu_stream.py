"""Partially resident (streamed) edge features: a cache budget smaller than h keeps a unit-aligned prefix of h and
recomputes the rest chunk by chunk inside every application (nnconv_apply_streamed).  The streamed h rows are the
bits the cached pass produces, so streamed and cached outputs differ only in the order of the fp32 scatter atomics.
Budgets are forced so that small graphs stream; the per-edge kernel matrices (which never stream) are switched off."""
import ctypes

import pytest
import torch

from oracle import nnconv_oracle as O
from tests.helpers import TOL, DenseNetLike, make_conv, oracle_stack_on_cuda, rel_err

pytestmark = pytest.mark.gpu

STREAM_TOL = 1e-5          # streamed vs cached, one application on the same input: scatter order only
# a chain of applications (residual steps, a whole KernelNN): an input that differs in the last fp32 bit can round to
# a neighbouring 16-bit Y operand in the next application
CHAIN_TOL = 1e-4


@pytest.fixture(scope='module')
def dev():
    assert torch.cuda.is_available()
    return torch.device('cuda:0')


@pytest.fixture(autouse=True)
def formulation_c(monkeypatch):
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_EDGE_KERNELS', 'off')
    monkeypatch.setattr(nn_conv, '_EF_WS_BYTES', 3 << 20)      # small chunks: many streamed chunks per application


def _cls():
    from graph_pde_b200.nn_conv import NNConv_old
    return NNConv_old


def _params(layers, w, seed=11):
    torch.manual_seed(seed)
    mlp = DenseNetLike(layers)
    lin = [m for m in mlp.layers if isinstance(m, torch.nn.Linear)]
    return ([l.weight.detach() for l in lin], [l.bias.detach() for l in lin], torch.randn(w, w) * 0.1,
            torch.randn(w) * 0.1)


def _ball(s, r, dev, seed=0):
    from graph_pde_b200 import graphs
    ei = graphs.ball_connectivity(s, r, dev, True)
    _, _, ea = graphs.darcy_sample(s, r, dev, seed=seed, edge_index=ei)
    return ei, ea


def _hub_graph(dev, N=300, E=5000, k_in=6, seed=5):
    """Unsorted edges, a hub source with 1500 out-edges (several chunks of 384 rows), duplicates, isolated nodes."""
    gen = torch.Generator().manual_seed(seed)
    src = torch.randint(0, N - 20, (E,), generator=gen)
    dst = torch.randint(10, N, (E,), generator=gen)
    src[:1500] = 7
    ei = torch.stack([src, dst])
    return ei.to(dev), torch.randn(E, k_in, generator=gen).to(dev)


def _stack(conv, x, ei, ea, T, budget, inputs=None):
    """T applications of one conv (one edge-feature cache) with the given budget: x_{k+1} = relu(conv(x_k)), or, with
    ``inputs``, conv(inputs[k]) -- the streamed run is fed the cached run's inputs so that a 16-bit rounding flip
    of the Y operand in one application does not propagate into the next.  Returns (outputs, inputs, chunk passes)."""
    from graph_pde_b200 import nn_conv
    conv.edge_feature_bytes = budget
    conv.invalidate()
    c0 = nn_conv.stats['streamed_chunk_passes']
    outs, ins = [], []
    with torch.no_grad():
        for k in range(T):
            if inputs is not None:
                x = inputs[k]
            ins.append(x)
            x = conv(x, ei, ea)
            outs.append(x)
            x = torch.relu(x)
    return outs, ins, nn_conv.stats['streamed_chunk_passes'] - c0


def _h_bytes(conv, ei, ea, n):
    from graph_pde_b200 import _lib, nn_conv
    plan = nn_conv.get_plan(ei, n, conv.flow)
    prep = conv._get_prepared(conv.precision)
    h_b, ws_b = ctypes.c_size_t(), ctypes.c_size_t()
    _lib.check(_lib.lib().nnconv_edge_features_sizes(plan.handle, prep.handle, 1 << 20, ctypes.byref(h_b),
                                                     ctypes.byref(ws_b)))
    return h_b.value


def _oracle_stack(x, ei, ea, ws, bs, root, bias, aggr, T, flow):
    if flow == 'target_to_source':
        ei = ei[[1, 0]]
    x = x.double().cpu()
    args = ([w.double() for w in ws], [b.double() for b in bs], None if root is None else root.double(),
            None if bias is None else bias.double())
    outs = []
    for _ in range(T):
        x = O.nnconv_forward(x, ei.cpu(), ea.double().cpu(), *args, aggr=aggr)
        outs.append(x)
        x = torch.relu(x)
    return outs


@pytest.mark.parametrize('flow', ['source_to_target', 'target_to_source'])
@pytest.mark.parametrize('root_bias', [True, False])
@pytest.mark.parametrize('aggr', ['mean', 'add'])
@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2'])
def test_streamed_matches_cached(dev, precision, aggr, root_bias, flow):
    """All T applications, budget 0 (every edge streamed) and half of h resident, against the cached run and the fp64
    oracle."""
    w, T = 32, 3
    ei, ea = _ball(20, 0.25, dev)
    ws, bs, root, bias = _params([6, 256, 256, w * w], w)
    if not root_bias:
        root = bias = None
    conv = make_conv(_cls(), ws, bs, root, bias, aggr, w, w, precision, dev)
    conv.flow = flow
    x0 = torch.randn(400, w, generator=torch.Generator().manual_seed(2)).to(dev)
    if aggr == 'add':
        x0 = x0 * 0.05
    ref, ins, n0 = _stack(conv, x0, ei, ea, T, None)
    assert n0 == 0
    hb = _h_bytes(conv, ei, ea, 400)
    exact = _oracle_stack(x0, ei, ea, ws, bs, root, bias, aggr, T, flow)
    for budget in (0, hb // 2):
        got, _, n = _stack(conv, x0, ei, ea, T, budget, ins)
        assert n >= T * 2, (budget, n)
        for k in range(T):
            assert rel_err(got[k], ref[k]) < STREAM_TOL, (budget, k, rel_err(got[k], ref[k]))
            assert rel_err(got[k], exact[k]) < TOL[precision], (budget, k, rel_err(got[k], exact[k]))


@pytest.mark.parametrize('chunk_bytes', [300007, 1000003, 2 << 30])
@pytest.mark.parametrize('precision', ['f16', 'f16x2'])
def test_hub_source_across_chunks(dev, monkeypatch, precision, chunk_bytes):
    """A hub source whose 1500 out-edges span several chunks (its Y is built in every launch that holds some of its
    units), chunk sizes that are not a multiple of 128 edges, and budgets 0 / mid / all-but-one-unit."""
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_EF_WS_BYTES', chunk_bytes)
    w, T = 64, 2
    ei, ea = _hub_graph(dev)
    ws, bs, root, bias = _params([6, 128, 64, w * w], w)
    conv = make_conv(_cls(), ws, bs, root, bias, 'mean', w, w, precision, dev)
    x0 = torch.randn(300, w, generator=torch.Generator().manual_seed(3)).to(dev)
    ref, ins, _ = _stack(conv, x0, ei, ea, T, None)
    hb = _h_bytes(conv, ei, ea, 300)
    for budget in (0, hb // 3, hb - 1):
        got, _, n = _stack(conv, x0, ei, ea, T, budget, ins)
        assert n >= T
        for k in range(T):
            assert rel_err(got[k], ref[k]) < STREAM_TOL, (budget, k)


def test_empty_graph_and_single_source(dev, monkeypatch):
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_EF_WS_BYTES', 300007)      # 256-edge chunks: the one source spans four
    w = 64
    ws, bs, root, bias = _params([6, 128, 128, w * w], w)
    conv = make_conv(_cls(), ws, bs, root, bias, 'mean', w, w, 'f16', dev)
    x0 = torch.randn(50, w, device=dev)
    ei = torch.zeros(2, 0, dtype=torch.int64, device=dev)
    ea = torch.zeros(0, 6, device=dev)
    ref, ins, _ = _stack(conv, x0, ei, ea, 1, None)
    got, _, n = _stack(conv, x0, ei, ea, 1, 0, ins)
    assert n == 0
    assert torch.equal(got[0], ref[0])
    gen = torch.Generator().manual_seed(1)
    ei = torch.stack([torch.full((1000,), 3, dtype=torch.int64), torch.randint(0, 50, (1000,), generator=gen)]).to(dev)
    ea = torch.randn(1000, 6, generator=gen).to(dev)
    ref, ins, _ = _stack(conv, x0, ei, ea, 2, None)
    got, _, n = _stack(conv, x0, ei, ea, 2, 0, ins)
    assert n >= 2 * 2
    for k in range(2):
        assert rel_err(got[k], ref[k]) < STREAM_TOL


@pytest.mark.parametrize('precision', ['f16', 'f16x2'])
def test_prefix_bits_equal_cached(dev, precision):
    """nnconv_edge_features_prefix writes exactly the first E_res rows of every panel of the cached h."""
    from graph_pde_b200 import _lib, nn_conv
    L = _lib.lib()
    w = 32
    ei, ea = _hub_graph(dev)
    ws, bs, root, bias = _params([6, 256, 256, w * w], w)
    conv = make_conv(_cls(), ws, bs, root, bias, 'mean', w, w, precision, dev)
    plan = nn_conv.get_plan(ei, 300, conv.flow)
    prep = conv._get_prepared(precision)
    ea32 = ea.contiguous().float()
    h = conv.edge_features(plan, prep, ea32)
    e_pad = (plan.E + 127) // 128 * 128
    panels = h.numel() // (e_pad * 128)
    for frac in (0.3, 0.7):
        e_res, hb, wsb, nch = ctypes.c_int64(), ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_int64()
        _lib.check(L.nnconv_stream_split(plan.handle, prep.handle, int(h.numel() * frac), 3 << 20, ctypes.byref(e_res),
                                         ctypes.byref(hb), ctypes.byref(wsb), ctypes.byref(nch)))
        E_res = e_res.value
        assert 0 < E_res < plan.E and nch.value >= 1
        hp = torch.empty(hb.value, dtype=torch.uint8, device=dev)
        ws_ef = torch.empty(64 << 20, dtype=torch.uint8, device=dev)
        _lib.check(L.nnconv_edge_features_prefix(plan.handle, prep.handle, nn_conv._ptr(ea32), E_res, nn_conv._ptr(hp),
                                                 nn_conv._ptr(ws_ef), ws_ef.numel(), nn_conv._stream_ptr(dev), None))
        torch.cuda.synchronize()
        r_pad = hb.value // (panels * 128)
        assert torch.equal(hp.view(panels, r_pad, 128)[:, :E_res], h.view(panels, e_pad, 128)[:, :E_res])


def test_no_fuse_option(dev):
    """The per-batch kernels (nnconv_set_option('no_fuse', 1)) over unit ranges with an edge base, PDL-pipelined and
    (no_pipe) in plain stream order."""
    from graph_pde_b200 import _lib
    w, T = 64, 2
    ei, ea = _hub_graph(dev)
    ws, bs, root, bias = _params([6, 128, 128, w * w], w)
    conv = make_conv(_cls(), ws, bs, root, bias, 'mean', w, w, 'f16', dev)
    x0 = torch.randn(300, w, device=dev)
    ref, ins, _ = _stack(conv, x0, ei, ea, T, None)
    for knobs in (('no_fuse',), ('no_fuse', 'no_pipe')):
        for k in knobs:
            _lib.set_option(k, 1)
        try:
            got, _, n = _stack(conv, x0, ei, ea, T, 0, ins)
            got2, _, _ = _stack(conv, x0, ei, ea, T, _h_bytes(conv, ei, ea, 300) // 2, ins)
        finally:
            for k in knobs:
                _lib.set_option(k, None)
        assert n >= T, knobs
        for k in range(T):
            assert rel_err(got[k], ref[k]) < STREAM_TOL, knobs
            assert rel_err(got2[k], ref[k]) < STREAM_TOL, knobs


def test_residual_step_chain(dev):
    w = 32
    ei, ea = _ball(20, 0.25, dev)
    ws, bs, root, bias = _params([6, 256, 256, w * w], w)
    conv = make_conv(_cls(), ws, bs, root, bias, 'mean', w, w, 'f16', dev)
    z0 = torch.randn(400, w, device=dev)

    def chain(budget, inputs=None):
        conv.edge_feature_bytes = budget
        conv.invalidate()
        z, ins, outs = z0, [], []
        with torch.no_grad():
            for k in range(3):
                z = inputs[k] if inputs is not None else z
                ins.append(z)
                z = conv.residual_step(z, ei, ea, relu_in=k > 0)
                outs.append(z)
        return outs, ins
    ref, ins = chain(None)
    got, _ = chain(0, ins)
    got_chain, _ = chain(0)
    for k in range(3):
        assert rel_err(got[k], ref[k]) < STREAM_TOL
        assert rel_err(got_chain[k], ref[k]) < CHAIN_TOL


def test_graphed_forward_streamed_kernelnn(dev):
    from graph_pde_b200 import nn_conv
    from graph_pde_b200.capture import GraphedForward
    from graph_pde_b200.models import KernelNN
    ei, ea = _ball(20, 0.25, dev)
    torch.manual_seed(0)
    model = KernelNN(32, 256, 4, 6, in_width=6, precision='f16').to(dev).eval()
    model.conv1.edge_feature_bytes = 1 << 20

    class D(object):
        pass
    d = D()
    d.x, d.edge_index, d.edge_attr = torch.randn(400, 6, device=dev), ei, ea
    with torch.no_grad():
        eager = model(d).clone()
    c0 = nn_conv.stats['streamed_chunk_passes']
    g = GraphedForward(model, d)
    assert nn_conv.stats['streamed_chunk_passes'] > c0
    out = g.replay()
    torch.cuda.synchronize()
    assert rel_err(out, eager) < CHAIN_TOL
    d.x.copy_(torch.randn(400, 6, device=dev))
    out = g.replay()
    with torch.no_grad():
        eager2 = model(d)
    assert rel_err(out, eager2) < CHAIN_TOL


def test_overflow_in_streamed_chunk_raises(dev):
    """Only the last edges (streamed: half of h is resident) leave the fp16 range: the resident prefix passes its check,
    the streamed application reports the overflow."""
    w = 32
    ei, ea0 = _ball(20, 0.25, dev)
    ws, bs, root, bias = _params([6, 256, 256, w * w], w)
    ws[1] = ws[1] * 200.0
    conv = make_conv(_cls(), ws, bs, root, bias, 'mean', w, w, 'f16', dev)
    conv.edge_feature_bytes = _h_bytes(conv, ei, ea0, 400) // 2
    x = torch.randn(400, w, device=dev)
    with torch.no_grad():
        conv(x, ei, ea0)                                 # in range: no report
    ea = ea0.clone()
    ea[-500:] *= 1e3                                     # with the hidden weights above: activations ~1e5
    with pytest.raises(FloatingPointError):
        with torch.no_grad():
            conv(x, ei, ea)


def test_autograd_with_streaming_raises(dev):
    w = 64
    ei, ea = _ball(20, 0.25, dev)
    ws, bs, root, bias = _params([6, 128, 128, w * w], w)
    conv = make_conv(_cls(), ws, bs, root, bias, 'mean', w, w, 'f16', dev)
    conv.edge_feature_bytes = 0
    x = torch.randn(400, w, device=dev, requires_grad=True)
    with pytest.raises(RuntimeError, match='training needs the whole h resident'):
        conv(x, ei, ea)


def test_auto_policy_streams_only_on_oom(dev, monkeypatch):
    from graph_pde_b200 import nn_conv
    w, T = 32, 2
    ei, ea = _ball(20, 0.25, dev)
    ws, bs, root, bias = _params([6, 256, 256, w * w], w)
    conv = make_conv(_cls(), ws, bs, root, bias, 'mean', w, w, 'f16', dev)
    x0 = torch.randn(400, w, device=dev)
    ref, ins, n = _stack(conv, x0, ei, ea, T, None)            # a normal allocation: no streaming
    assert n == 0
    assert all(isinstance(v[0], torch.Tensor) for v in conv._h_cache.values())
    hb = _h_bytes(conv, ei, ea, 400)
    real_empty = torch.empty

    def empty_oom(*args, **kw):
        if args and args[0] == hb:                         # the whole h (and a prefix as large as it) does not fit
            raise torch.cuda.OutOfMemoryError('simulated: h does not fit')
        return real_empty(*args, **kw)
    monkeypatch.setattr(torch, 'empty', empty_oom)
    got, _, n = _stack(conv, x0, ei, ea, T, None, ins)
    monkeypatch.setattr(torch, 'empty', real_empty)
    assert n >= T
    for k in range(T):
        assert rel_err(got[k], ref[k]) < STREAM_TOL


def test_darcy241_f16x2_full_stack_streamed(dev, monkeypatch):
    """The fp32-grade mode at the headline size: 241x241, r=0.05 (E = 24,557,297), w=64, ker_width=1024, T=6, f16x2
    (4 KB of edge features per edge, 94 GiB: more than an 80 GB H100 holds) with a 40 GB resident prefix, against the
    fp32 reference ops on the GPU."""
    from graph_pde_b200 import graphs, nn_conv
    monkeypatch.setattr(nn_conv, '_EF_WS_BYTES', 2 << 30)
    s, r, T, w = 241, 0.05, 6, 64
    ei = graphs.ball_connectivity(s, r, dev, True)
    _, _, ea = graphs.darcy_sample(s, r, dev, seed=3, edge_index=ei)
    assert ei.size(1) == 24557297
    ws, bs, root, bias = O.reference_init(w, w, [6, 1024, 1024, w * w], seed=0)
    torch.manual_seed(3)
    x0 = torch.randn(s * s, w, device=dev)
    conv = make_conv(_cls(), ws, bs, root, bias, 'mean', w, w, 'f16x2', dev)
    conv.edge_feature_bytes = 40 << 30
    c0 = nn_conv.stats['streamed_chunk_passes']
    got = []
    x = x0
    with torch.no_grad():
        for _ in range(T):
            x = torch.relu(conv(x, ei, ea))
            got.append(x)
    assert nn_conv.stats['streamed_chunk_passes'] > c0
    conv.invalidate()
    torch.cuda.empty_cache()
    dws, dbs = [v.to(dev) for v in ws], [v.to(dev) for v in bs]
    ref = oracle_stack_on_cuda(x0, ei, ea, dws, dbs, root.to(dev), bias.to(dev), T, edge_chunk=1 << 16)
    errs = [rel_err(got[k], ref[k]) for k in range(T)]
    assert max(errs) < TOL['f16x2'], errs
