"""The diagonal-kernel NNConv on the H100: parity with the reference's outputs (g8) and the fp64 oracle at every
precision and aggregation, exact integer probes whose outputs, argmax and gradients must equal fp64 autograd bit for
bit (add, max) or within a per-node bound (mean), random-data gradients, and a CUDA-graph replay of the forward.

Why the probes are exact: x, edge_attr, the output gradient and every weight and bias of the edge network are small
integers (weights in {-1, 0, 1}).  Every activation of the edge network is an integer below 2^8, so bf16, fp16 and the
f16x2 pairs hold it exactly; d_e, the messages x * d, and every fp32 sum of the forward and the backward stay below 2^24
(the largest, dW_L = dd^T h, is at most E * 4 * 3 * 64 * 8 < 2^24 for the graphs here).  So no operation rounds, in any
order, and the library must produce the fp64 result exactly.
"""
import pytest
import torch

from graph_pde_b200 import nn_conv
from graph_pde_b200.nn_conv import DiagNNConv
from oracle import golden
from tests import diag_oracle as D
from tests.helpers import TOL

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
PRECS = ['f16', 'bf16', 'f16x2', 'fp32']
C, KIN, WIDTH = 64, 3, 64


def _graph(n=300, e=6000, seed=0):
    """Random graph with a hub source (node 0: 1/6 of the edges, > 128 so it spans many tiles), nodes 0..4 without
    in-edges and duplicate edges."""
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n, (e,), generator=g)
    dst = torch.randint(5, n, (e,), generator=g)
    src[: e // 6] = 0
    src[10:20], dst[10:20] = src[9], dst[9]
    perm = torch.randperm(e, generator=g)
    return torch.stack([src[perm], dst[perm]])


def _mlp():
    return torch.nn.Sequential(torch.nn.Linear(KIN, WIDTH), torch.nn.ReLU(), torch.nn.Linear(WIDTH, C))


def _probe_layers(seed):
    g = torch.Generator().manual_seed(seed)
    w1 = torch.randint(-1, 2, (WIDTH, KIN), generator=g).float()
    b1 = torch.randint(-1, 3, (WIDTH,), generator=g).float()
    w2 = torch.randint(-1, 2, (C, WIDTH), generator=g).float() * (torch.rand(C, WIDTH, generator=g) < 0.25)
    b2 = torch.randint(-2, 3, (C,), generator=g).float()
    return [(w1, b1), (w2, b2)]


def _conv(layers, aggr, precision, root, bias, flow='source_to_target'):
    conv = DiagNNConv(C, C, _mlp(), aggr=aggr, precision=precision, flow=flow,
                      root_weight=root is not None, bias=bias is not None)
    with torch.no_grad():       # after the constructor, whose reset_parameters re-initialises nn
        for lin, (w, b) in zip([conv.nn[0], conv.nn[2]], layers):
            lin.weight.copy_(w)
            lin.bias.copy_(b)
        if root is not None:
            conv.root.copy_(root)
        if bias is not None:
            conv.bias.copy_(bias)
    return conv.to(DEV)


def _ref_layers(layers):
    return [w.double() for w, _ in layers], [b.double() for _, b in layers]


@pytest.mark.parametrize('precision', PRECS)
def test_g8_parity(precision):
    """Every case of the reference's own outputs with 64 channels, every aggregation, root / bias on and off."""
    rec = golden.load(golden_path())
    ei = torch.from_numpy(rec['edge_index']).to(DEV)
    ea = torch.from_numpy(rec['edge_attr']).to(DEV)
    x = torch.from_numpy(rec['x']).to(DEV)
    for i in range(int(rec['n_cases'])):
        aggr, rw, bs, c = [str(v) for v in rec['c%d_case' % i]]
        if int(c) != C:
            continue
        p = 'c%d_' % i
        layers = [(torch.from_numpy(rec[p + 'sd_nn.%d.weight' % l]), torch.from_numpy(rec[p + 'sd_nn.%d.bias' % l]))
                  for l in (0, 2)]
        root = torch.from_numpy(rec[p + 'sd_root']) if rw == 'True' else None
        bias = torch.from_numpy(rec[p + 'sd_bias']) if bs == 'True' else None
        conv = _conv(layers, aggr, precision, root, bias)
        with torch.no_grad():
            out = conv(x, ei, ea)
        ref = torch.from_numpy(rec[p + 'out']).to(DEV)
        err = ((out - ref).abs().max() / ref.abs().max()).item()
        assert err < TOL[precision], (i, aggr, rw, bs, err)


def test_g8_one_dimensional_x():
    rec = golden.load(golden_path())
    i = int(rec['n_cases']) - 1
    p = 'c%d_' % i
    assert str(rec[p + 'case'][3]) == '1'
    conv = DiagNNConv(1, 1, torch.nn.Sequential(torch.nn.Linear(KIN, WIDTH), torch.nn.ReLU(), torch.nn.Linear(WIDTH, 1)),
                      aggr='mean', precision='fp32')
    conv.load_state_dict({k[len(p) + 3:]: torch.from_numpy(v) for k, v in rec.items() if k.startswith(p + 'sd_')})
    conv = conv.to(DEV)
    with torch.no_grad():
        out = conv(torch.from_numpy(rec['x1']).to(DEV), torch.from_numpy(rec['edge_index']).to(DEV),
                   torch.from_numpy(rec['edge_attr']).to(DEV))
    ref = torch.from_numpy(rec[p + 'out']).to(DEV)
    assert out.shape == ref.shape
    assert ((out - ref).abs().max() / ref.abs().max()).item() < TOL['fp32']


def golden_path():
    import os
    return os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'g8_diag_nnconv.npz')


@pytest.mark.parametrize('precision', PRECS)
@pytest.mark.parametrize('aggr', ['add', 'mean', 'max'])
@pytest.mark.parametrize('flow', ['source_to_target', 'target_to_source'])
def test_random_forward_and_gradients(precision, aggr, flow):
    """Random data: out within TOL of the fp64 oracle; every gradient within the backward's fp32 tolerance of fp64
    autograd routed by the library's own argmax (so a near-tie does not flip a winner between the two)."""
    g = torch.Generator().manual_seed(11)
    ei = _graph(seed=1)
    e = ei.size(1)
    layers = [(torch.randn(WIDTH, KIN, generator=g) * 0.5, torch.randn(WIDTH, generator=g) * 0.1),
              (torch.randn(C, WIDTH, generator=g) * 0.2, torch.randn(C, generator=g) * 0.1)]
    root, bias = torch.randn(C, C, generator=g) * 0.1, torch.randn(C, generator=g) * 0.1
    x = torch.randn(300, C, generator=g)
    ea = torch.randn(e, KIN, generator=g)
    conv = _conv(layers, aggr, precision, root, bias, flow)
    xd, ead = x.to(DEV).requires_grad_(), ea.to(DEV).requires_grad_()
    out = conv(xd, ei.to(DEV), ead)
    gout = torch.randn(300, C, generator=g)
    out.backward(gout.to(DEV))
    # fp64 reference, the max routed by the library's argmax
    ws, bs = _ref_layers(layers)
    ws = [w.requires_grad_() for w in ws]
    bs = [b.requires_grad_() for b in bs]
    xr, ear = x.double().requires_grad_(), ea.double().requires_grad_()
    rr, br = root.double().requires_grad_(), bias.double().requires_grad_()
    am = None
    if aggr == 'max':
        _, am_lib = conv._apply_impl(conv._tstate.plan, conv._tstate.feats, xd.detach())
        am = am_lib.long().cpu()
        _, am_ref = D.nnconv_diag_forward(x.double(), ei, ea.double(), [w.detach() for w in ws], [b.detach() for b in bs],
                                          flow=flow, aggr='max')
        assert (am != am_ref).float().mean().item() < (1e-3 if precision in ('fp32', 'f16x2') else 5e-2)
    ref, _ = D.nnconv_diag_forward(xr, ei, ear, ws, bs, rr, br, aggr, flow, argmax=am)
    ref.backward(gout.double())
    assert ((out.detach().cpu().double() - ref.detach()).abs().max() / ref.abs().max()).item() < TOL[precision]
    pairs = [(xd.grad, xr.grad), (ead.grad, ear.grad), (conv.root.grad, rr.grad), (conv.bias.grad, br.grad),
             (conv.nn[0].weight.grad, ws[0].grad), (conv.nn[0].bias.grad, bs[0].grad),
             (conv.nn[2].weight.grad, ws[1].grad), (conv.nn[2].bias.grad, bs[1].grad)]
    tol = 1e-4 if precision in ('fp32', 'f16x2') else 3e-2
    for k, (a, b) in enumerate(pairs):
        err = ((a.cpu().double() - b).abs().max() / b.abs().max().clamp(min=1e-30)).item()
        assert err < tol, (k, err)


@pytest.mark.parametrize('precision', PRECS)
@pytest.mark.parametrize('aggr', ['add', 'max', 'mean'])
@pytest.mark.parametrize('T', [1, 2, 6])
@pytest.mark.parametrize('flow', ['source_to_target', 'target_to_source'])
def test_exact_probe_forward_backward(precision, aggr, T, flow):
    """Integer probe, T applications of one conv sharing ONE edge-network pass: out, argmax and every gradient equal
    fp64 autograd exactly (add, max); mean within 2^-20 of each node's largest term.  target_to_source reads the same
    edge_index the other way round: the hub is then a target, and the nodes 0..4 have no out-edges instead."""
    g = torch.Generator().manual_seed(5 + T)
    ei = _graph(seed=2)
    e = ei.size(1)
    layers = _probe_layers(7)
    root = torch.randint(-1, 2, (C, C), generator=g).float()
    bias = torch.randint(-2, 3, (C,), generator=g).float()
    xs = [torch.randint(-4, 5, (300, C), generator=g).float() for _ in range(T)]
    ea = torch.randint(-2, 3, (e, KIN), generator=g).float()
    gouts = [torch.randint(-3, 4, (300, C), generator=g).float() for _ in range(T)]
    conv = _conv(layers, aggr, precision, root, bias, flow)
    ead = ea.to(DEV).requires_grad_()
    eid = ei.to(DEV)            # one edge_index for every application, as KernelNN passes it
    xds = [x.to(DEV).requires_grad_() for x in xs]
    outs = [conv(xd, eid, ead) for xd in xds]
    mlp_before = nn_conv.stats['mlp_backwards']
    sum((o * gg.to(DEV)).sum() for o, gg in zip(outs, gouts)).backward()
    assert nn_conv.stats['mlp_backwards'] - mlp_before == 1      # the T applications share one edge-network pass
    ws, bs = _ref_layers(layers)
    ws = [w.requires_grad_() for w in ws]
    bs = [b.requires_grad_() for b in bs]
    ear = ea.double().requires_grad_()
    rr, br = root.double().requires_grad_(), bias.double().requires_grad_()
    xrs = [x.double().requires_grad_() for x in xs]
    refs = [D.nnconv_diag_forward(xr, ei, ear, ws, bs, rr, br, aggr, flow) for xr in xrs]
    sum((r * gg.double()).sum() for (r, _), gg in zip(refs, gouts)).backward()

    def same(a, b, what, per_node=True):
        a = a.detach().cpu().double()
        if aggr == 'mean':
            # mean scales each message by 1 / deg, which rounds: a node's rows sum ~20 rounded terms, a parameter
            # gradient sums one per edge (6000), so its bound is 2^4 wider
            bound = 2 ** (-20 if per_node else -16)
            assert (a - b).abs().max().item() <= bound * max(b.abs().max().item(), 1.0), what
        else:
            assert torch.equal(a, b.detach()), (what, (a - b).abs().max().item())

    for t in range(T):
        same(outs[t], refs[t][0], 'out %d' % t)
        same(xds[t].grad, xrs[t].grad, 'dx %d' % t)
        if aggr == 'max':
            _, am = conv._apply_impl(conv._tstate.plan, conv._tstate.feats, xds[t].detach())
            assert torch.equal(am.long().cpu(), refs[t][1]), 'argmax %d' % t
            if flow == 'source_to_target':
                assert (refs[t][1][:5] == -1).all()
    for a, b, what in [(ead.grad, ear.grad, 'edge_attr'), (conv.root.grad, rr.grad, 'root'), (conv.bias.grad, br.grad, 'bias'),
                       (conv.nn[0].weight.grad, ws[0].grad, 'W1'), (conv.nn[0].bias.grad, bs[0].grad, 'b1'),
                       (conv.nn[2].weight.grad, ws[1].grad, 'W2'), (conv.nn[2].bias.grad, bs[1].grad, 'b2')]:
        same(a, b, what, per_node=False)


@pytest.mark.parametrize('precision', PRECS)
def test_chunked_build_matches_one_chunk(precision, monkeypatch):
    """d built in many chunks (a small workspace) equals d built in one chunk, and the exact probe's output."""
    g = torch.Generator().manual_seed(9)
    ei = _graph(n=2000, e=60000, seed=3)
    layers = _probe_layers(3)
    x = torch.randint(-4, 5, (2000, C), generator=g).float()
    ea = torch.randint(-2, 3, (ei.size(1), KIN), generator=g).float()
    outs = []
    for ws_bytes in (1 << 30, 1 << 20):
        monkeypatch.setattr(nn_conv, '_DIAG_WS_BYTES', ws_bytes)
        conv = _conv(layers, 'add', precision, None, None)
        before = nn_conv.stats['launches']
        with torch.no_grad():
            outs.append(conv(x.to(DEV), ei.to(DEV), ea.to(DEV)).cpu())
        assert nn_conv.stats['launches'] > before
    ws, bs = _ref_layers(layers)
    ref, _ = D.nnconv_diag_forward(x.double(), ei, ea.double(), ws, bs, aggr='add')
    assert torch.equal(outs[0].double(), ref) and torch.equal(outs[1].double(), ref)


def test_graphed_forward_replay():
    from graph_pde_b200 import GraphedForward
    g = torch.Generator().manual_seed(4)
    ei = _graph(seed=4).to(DEV)
    layers = _probe_layers(4)
    conv = _conv(layers, 'max', 'f16', None, None)
    x = torch.randint(-4, 5, (300, C), generator=g).float().to(DEV)
    ea = torch.randint(-2, 3, (ei.size(1), KIN), generator=g).float().to(DEV)
    gf = GraphedForward(conv, x, ei, ea)
    x2 = torch.randint(-4, 5, (300, C), generator=g).float().to(DEV)
    x.copy_(x2)
    out = gf.replay().clone()
    with torch.no_grad():
        ref = conv(x2, ei, ea)
    assert torch.equal(out, ref)


@pytest.mark.parametrize('precision', PRECS)
def test_frozen_edge_network_skips_grad_d(precision):
    """With neither the edge network nor edge_attr requiring a gradient, no grad_d is allocated and no edge-network pass
    runs; the gradients of x, root and bias are still exact."""
    g = torch.Generator().manual_seed(21)
    ei = _graph(seed=5)
    layers = _probe_layers(5)
    root = torch.randint(-1, 2, (C, C), generator=g).float()
    bias = torch.randint(-2, 3, (C,), generator=g).float()
    conv = _conv(layers, 'add', precision, root, bias)
    for p in conv.nn.parameters():
        p.requires_grad_(False)
    x = torch.randint(-4, 5, (300, C), generator=g).float()
    ea = torch.randint(-2, 3, (ei.size(1), KIN), generator=g).float()
    gout = torch.randint(-3, 4, (300, C), generator=g).float()
    xd = x.to(DEV).requires_grad_()
    mlp_before = nn_conv.stats['mlp_backwards']
    for _ in range(2):
        xd.grad = None
        conv.root.grad = conv.bias.grad = None
        (conv(xd, ei.to(DEV), ea.to(DEV)) * gout.to(DEV)).sum().backward()
        assert conv._tstate.dd is None and conv._tstate.token is None
    assert nn_conv.stats['mlp_backwards'] == mlp_before
    ws, bs = _ref_layers(layers)
    xr, rr, br = x.double().requires_grad_(), root.double().requires_grad_(), bias.double().requires_grad_()
    ref, _ = D.nnconv_diag_forward(xr, ei, ea.double(), ws, bs, rr, br, 'add')
    (ref * gout.double()).sum().backward()
    for a, b in ((xd.grad, xr.grad), (conv.root.grad, rr.grad), (conv.bias.grad, br.grad)):
        assert torch.equal(a.cpu().double(), b)


def test_x_not_16_byte_aligned():
    """x starting one float into its storage: the application falls back to 4-byte accesses and still matches."""
    g = torch.Generator().manual_seed(22)
    ei = _graph(seed=6).to(DEV)
    conv = _conv(_probe_layers(6), 'add', 'f16', None, None)
    x = torch.randint(-4, 5, (300, C), generator=g).float().to(DEV)
    ea = torch.randint(-2, 3, (ei.size(1), KIN), generator=g).float().to(DEV)
    buf = torch.empty(300 * C + 1, device=DEV)
    xm = buf[1:].view(300, C)
    xm.copy_(x)
    assert xm.is_contiguous() and xm.data_ptr() % 16 != 0
    with torch.no_grad():
        assert torch.equal(conv(xm, ei, ea), conv(x, ei, ea))


def test_darcy241_exact_application_chunked_build():
    """One application on the 241^2, r = 0.05 mesh (24.6 M edges) with an exact probe: d is built in several chunks and
    out equals the fp64 result, computed on the GPU in edge chunks."""
    from graph_pde_b200 import _lib, graphs
    import ctypes
    ei = graphs.ball_connectivity(241, 0.05, device=DEV)
    e = ei.size(1)
    src, dst = ei
    ea = torch.stack([((src * 7 + dst * 13) % 5 - 2), ((src * 3 + dst * 11) % 5 - 2), ((src + dst * 5) % 5 - 2)], 1).float()
    g = torch.Generator().manual_seed(23)
    layers = _probe_layers(8)
    x = torch.randint(-4, 5, (241 * 241, C), generator=g).float().to(DEV)
    conv = _conv(layers, 'add', 'f16', None, None)
    with torch.no_grad():
        out = conv(x, ei, ea)
    st = next(iter(conv._d_cache.values()))
    d_b, ws_b = ctypes.c_size_t(), ctypes.c_size_t()
    _lib.check(_lib.lib().nnconv_diag_sizes(nn_conv.get_plan(ei, x.size(0)).handle, st.prepared.handle,
                                            nn_conv._DIAG_WS_BYTES, ctypes.byref(d_b), ctypes.byref(ws_b)))
    assert ws_b.value < e * 128 // 2          # the chunk holds less than half of the mesh's h: several chunks
    del st
    ws = [w.double().to(DEV) for w, _ in layers]
    bs = [b.double().to(DEV) for _, b in layers]
    ref = torch.zeros(x.size(0), C, dtype=torch.float64, device=DEV)
    step = 1 << 22
    for s0 in range(0, e, step):
        sl = slice(s0, min(s0 + step, e))
        dref = D.O.dense_net(ea[sl].double(), ws, bs)
        ref.index_add_(0, dst[sl], x[src[sl]].double() * dref)
    assert torch.equal(out.double(), ref)


def test_graphed_train_step_replay_equals_eager():
    """A KernelNN-shaped model around one shared DiagNNConv (T = 3), trained by GraphedTrainStep and eagerly on two
    copies: losses and parameters agree step by step, and an eager forward after the replays sees the replayed
    parameters (the caches the capture and the replays left behind are dropped)."""
    import os
    import numpy as np
    import torch.nn.functional as F
    from graph_pde_b200 import GraphedTrainStep
    from tests.helpers import GOLDEN, ei64, rel_err, t
    gd = np.load(os.path.join(GOLDEN, 'g2_cfg1_ball16.npz'))
    x, ei, ea = t(gd['node_x']).to(DEV), ei64(gd['edge_index']).to(DEV), t(gd['edge_attr']).to(DEV)
    y = torch.randn(x.size(0), 1, generator=torch.Generator().manual_seed(0)).to(DEV)

    class Net(torch.nn.Module):
        def __init__(self, precision):
            super().__init__()
            self.fc1 = torch.nn.Linear(x.size(1), C)
            mlp = torch.nn.Sequential(torch.nn.Linear(ea.size(1), WIDTH), torch.nn.ReLU(), torch.nn.Linear(WIDTH, C))
            self.conv = DiagNNConv(C, C, mlp, aggr='mean', precision=precision)
            self.fc2 = torch.nn.Linear(C, 1)

        def forward(self, xin, eain):
            h = self.fc1(xin)
            for _ in range(3):
                h = F.relu(self.conv(h, ei, eain))
            return self.fc2(h)

    for precision, tol in (('f16x2', 1e-4), ('fp32', 1e-4), ('f16', 3e-3)):
        torch.manual_seed(0)
        model_e, model_g = Net(precision).to(DEV), Net(precision).to(DEV)
        model_g.load_state_dict(model_e.state_dict())
        opt_e = torch.optim.Adam(model_e.parameters(), lr=1e-3, capturable=True)
        opt_g = torch.optim.Adam(model_g.parameters(), lr=1e-3, capturable=True)
        xg, eag, yg = x.clone(), ea.clone(), y.clone()
        step = GraphedTrainStep(lambda a, b, c: F.mse_loss(model_g(a, b), c), model_g, opt_g, xg, eag, yg)
        for i in range(5):
            opt_e.zero_grad(set_to_none=True)
            loss_e = F.mse_loss(model_e(x, ea), y)
            loss_e.backward()
            opt_e.step()
            loss_g = step.replay()
            assert rel_err(loss_g, loss_e.detach()) < tol, (precision, i, float(loss_g), float(loss_e))
            for (name, pg), pe in zip(model_g.named_parameters(), model_e.parameters()):
                assert rel_err(pg, pe) < tol, (precision, i, name)
        with torch.no_grad():
            assert rel_err(model_g(x, ea), model_e(x, ea)) < tol, precision
