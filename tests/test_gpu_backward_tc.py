"""GPU: the tensor-core backward (csrc/backward_tc.cu, csrc/gemm_tn.cu) -- unit tests of its GEMM building blocks
against torch, and gradient parity of the whole op against autograd through the oracle (fp64 on the CPU for small
graphs, fp32 torch ops on the GPU at BASELINE config-2 size).  pytest -m gpu."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import nnconv_oracle as O
from tests.helpers import DenseNetLike, emulated_nnconv_forward, make_conv

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
# stated gradient tolerances, max|g - ref| / max|ref| per tensor: against autograd through a forward that rounds
# where the kernels round (tests/helpers.py explains why), and -- loose -- against the exact fp64 oracle
GTOL = {'f16': 3e-3, 'bf16': 3e-2}
GTOL_EXACT = 8e-2


def _relerr(got, ref):
    ref = ref.detach().double().cpu()
    return float((got.detach().double().cpu() - ref).abs().max() / ref.abs().max().clamp(min=1e-30))


@pytest.mark.parametrize('prec,dt', [('f16', torch.float16), ('bf16', torch.bfloat16)])
@pytest.mark.parametrize('R,M,N', [(5000, 1024, 1024), (777, 128, 64), (64, 64, 64), (100000, 256, 64), (3001, 192, 320)])
def test_gemm_tn_matches_torch(prec, dt, R, M, N):
    """C += alpha * A^T B with both operands taken row-major (MN-major wgmma descriptors), split over the rows."""
    from graph_pde_b200 import _lib
    L = _lib.lib()
    _lib.check(L.nnconv_init())
    g = torch.Generator(device='cpu').manual_seed(R + M + N)
    lda, ldb = ((M + 63) // 64) * 64 + 64, ((N + 63) // 64) * 64
    A = (torch.randn(R, lda, generator=g) * 0.5).to(DEV).to(dt)
    B = (torch.randn(R, ldb, generator=g) * 0.5).to(DEV).to(dt)
    C0 = torch.randn(M, N, generator=g).to(DEV)
    C = C0.clone()
    _lib.check(L.nnconv_gemm_tn_16b(_lib.PREC[prec], A.data_ptr(), lda, B.data_ptr(), ldb, R, M, N, C.data_ptr(), N, 0.5,
                                    torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    ref = C0.double() + 0.5 * (A[:, :M].double().t() @ B[:, :N].double())
    assert _relerr(C, ref) < 1e-4, (R, M, N)


@pytest.mark.parametrize('prec,dt', [('f16', torch.float16), ('bf16', torch.bfloat16)])
def test_gemm_mask_and_f32_epilogues(prec, dt):
    from graph_pde_b200 import _lib
    L = _lib.lib()
    _lib.check(L.nnconv_init())
    g = torch.Generator(device='cpu').manual_seed(3)
    M, K, N = 1000, 256, 128
    A = (torch.randn(M, K, generator=g) * 0.3).to(DEV).to(dt)
    B = (torch.randn(N, K, generator=g) * 0.3).to(DEV).to(dt)
    act = torch.relu(torch.randn(M, N, generator=g)).to(DEV).to(dt)          # ~half zeros
    st = torch.cuda.current_stream().cuda_stream
    ref = A.double() @ B.double().t()
    C = torch.zeros(M, N, device=DEV, dtype=dt)
    _lib.check(L.nnconv_gemm_16b_ex(_lib.PREC[prec], A.data_ptr(), M, K, B.data_ptr(), N, None, 0, C.data_ptr(), N,
                                    act.data_ptr(), N, 0, st))
    torch.cuda.synchronize()
    assert _relerr(C, ref * (act > 0)) < (4e-3 if prec == 'f16' else 3e-2)
    C32 = torch.zeros(M, N, device=DEV)
    _lib.check(L.nnconv_gemm_16b_ex(_lib.PREC[prec], A.data_ptr(), M, K, B.data_ptr(), N, None, 0, C32.data_ptr(), N, None,
                                    0, 1, st))
    torch.cuda.synchronize()
    assert _relerr(C32, ref) < 1e-4


def _graph(gen, N, E, hub=False):
    src = torch.randint(0, N - 5, (E,), generator=gen)
    dst = torch.randint(2, N, (E,), generator=gen)
    if hub:
        src[:300] = 3
    order = torch.argsort(src, stable=True) if not hub else torch.arange(E)
    return torch.stack([src[order], dst[order]])


@pytest.mark.parametrize('layers,cin,aggr,rw,bs,prec', [
    ([6, 64, 64, 64 * 64], 64, 'mean', True, True, 'f16'),
    ([6, 64, 64, 64 * 64], 64, 'add', True, True, 'bf16'),
    ([6, 128, 32 * 64], 32, 'mean', False, False, 'f16'),            # 2-layer MLP (MGKN down/up), in < out
    ([4, 256, 320, 64 * 64], 64, 'mean', True, False, 'f16'),        # k_in = 4, Kp = 320: odd number of 64-chunks, k block 64
    ([6, 16, 32, 24, 64 * 64], 64, 'add', False, True, 'f16'),       # 4-layer MLP, widths padded to 64
])
def test_tc_backward_matches_autograd_through_oracle(layers, cin, aggr, rw, bs, prec):
    from graph_pde_b200.nn_conv import NNConv_old, stats
    cout = 64
    gen = torch.Generator().manual_seed(17)
    N, E = 150, 2500
    ei = _graph(gen, N, E, hub=True)                 # unsorted sources + a hub with several tiles
    ea = torch.randn(E, layers[0], generator=gen)
    x = torch.randn(N, cin, generator=gen)
    torch.manual_seed(3)
    mlp = DenseNetLike(layers)
    lin = [m for m in mlp.layers if isinstance(m, torch.nn.Linear)]
    ws = [l.weight.detach().clone() for l in lin]
    bsl = [l.bias.detach().clone() for l in lin]
    root = torch.randn(cin, cout) * 0.2 if rw else None
    bias = torch.randn(cout) * 0.2 if bs else None
    gout = torch.randn(N, cout, generator=gen) * 1e-3              # small gradients: exercises the power-of-two scaling
    def reference(fwd):
        leaves = [t.double().requires_grad_(True) for t in [x] + ws + bsl + ([root] if rw else []) + ([bias] if bs else [])]
        xr, wr, br = leaves[0], leaves[1:1 + len(ws)], leaves[1 + len(ws):1 + 2 * len(ws)]
        rest = leaves[1 + 2 * len(ws):]
        rr = rest.pop(0) if rw else None
        bbr = rest.pop(0) if bs else None
        (fwd(xr, wr, br, rr, bbr) * gout.double()).sum().backward()
        g = {'x': xr.grad}
        for i in range(len(ws)):
            g['W%d' % i], g['b%d' % i] = wr[i].grad, br[i].grad
        if rw:
            g['root'] = rr.grad
        if bs:
            g['bias'] = bbr.grad
        return g
    ref_exact = reference(lambda xr, wr, br, rr, bbr: O.nnconv_forward(xr, ei, ea.double(), wr, br, rr, bbr, aggr, cin, cout))
    ref_emul = reference(lambda xr, wr, br, rr, bbr: emulated_nnconv_forward(xr, ei, ea.double(), wr, br, rr, bbr, aggr, prec))
    conv = make_conv(NNConv_old, ws, bsl, root, bias, aggr, cin, cout, prec, DEV)
    n0 = stats.get('mlp_backwards', 0)
    xd = x.to(DEV).requires_grad_(True)
    out = conv(xd, ei.to(DEV), ea.to(DEV))
    (out * gout.to(DEV)).sum().backward()
    assert stats.get('mlp_backwards', 0) == n0 + 1       # the tensor-core path ran
    got = {'x': xd.grad}
    lin_d = [m for m in conv.nn.layers if isinstance(m, torch.nn.Linear)]
    for i, l in enumerate(lin_d):
        got['W%d' % i], got['b%d' % i] = l.weight.grad, l.bias.grad
    if rw:
        got['root'] = conv.root.grad
    if bs:
        got['bias'] = conv.bias.grad
    errs = {k: _relerr(got[k], ref_emul[k]) for k in got}
    errs_exact = {k: _relerr(got[k], ref_exact[k]) for k in got}
    bad = {k: v for k, v in errs.items() if not v < GTOL[prec]}
    bad_exact = {k: v for k, v in errs_exact.items() if not v < GTOL_EXACT}
    assert not bad and not bad_exact, (bad, bad_exact, errs, errs_exact)


def test_kernelnn_training_step_tc(dev=DEV):
    """KernelNN applies ONE conv T times: every application's backward runs on the tensor cores and the hidden
    layers are differentiated ONCE for all T (UAI1_full_resolution.py:29-30, loss.backward() :266).  Reference:
    autograd (fp64) through the mask-consistent forward, with the node-level ReLUs evaluated at the CUDA path's own
    conv outputs (same masks as the torch ReLUs that follow the CUDA conv)."""
    from graph_pde_b200.models import KernelNN
    from graph_pde_b200.nn_conv import stats
    gen = torch.Generator().manual_seed(5)
    s, r, w, kw, T = 12, 0.3, 64, 128, 4
    ei = torch.from_numpy(O.ball_connectivity(s, r))
    theta = np.random.RandomState(0).randn(s * s)
    ea = torch.from_numpy(O.ball_edge_attr(O.square_grid(s), ei.numpy(), theta))
    node_x = torch.randn(s * s, 6, generator=gen)
    y = torch.randn(s * s, 1, generator=gen)
    torch.manual_seed(0)
    model = KernelNN(w, kw, T, 6, in_width=6, precision='f16').to(dev)
    st = {k: v.detach().cpu().double() for k, v in model.state_dict().items()}

    class D(object):
        pass
    d = D()
    d.x, d.edge_index, d.edge_attr = node_x.to(dev), ei.to(dev), ea.to(dev)
    conv_outs = []
    hook = model.conv1.register_forward_hook(lambda m, i, o: conv_outs.append(o.detach().double().cpu()))
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    n_mlp, n_app = stats.get('mlp_backwards', 0), stats.get('backwards', 0)
    loss = torch.nn.functional.mse_loss(model(d), y.to(dev))
    loss.backward()
    hook.remove()
    assert stats.get('mlp_backwards', 0) == n_mlp + 1 and stats.get('backwards', 0) == n_app + T
    # reference
    leaves = {k: v.clone().requires_grad_(True) for k, v in st.items()}
    ws, bs = O.mlp_params_from_state(leaves, 'conv1.nn.')
    xr = torch.nn.functional.linear(node_x.double(), leaves['fc1.weight'], leaves['fc1.bias'])
    for k in range(T):
        o = emulated_nnconv_forward(xr, ei, ea.double(), ws, bs, leaves['conv1.root'], leaves['conv1.bias'], 'mean', 'f16')
        xr = torch.relu(o + (conv_outs[k] - o).detach())
    out_ref = torch.nn.functional.linear(xr, leaves['fc2.weight'], leaves['fc2.bias'])
    torch.nn.functional.mse_loss(out_ref, y.double()).backward()
    errs = {k: _relerr(p.grad, leaves[k].grad) for k, p in model.named_parameters()}
    bad = {k: v for k, v in errs.items() if not v < 5e-3}
    assert not bad, (bad, errs)
    opt.step()
    # a second step re-prepares the weights, recomputes the edge features and still works
    opt.zero_grad()
    loss2 = torch.nn.functional.mse_loss(model(d), y.to(dev))
    loss2.backward()
    assert stats.get('mlp_backwards', 0) == n_mlp + 2
    assert bool(torch.isfinite(loss2))


def test_tc_backward_config2_size():
    """BASELINE config-2 size graph (85x85, r=0.10, E = 1,466,497), w=64, ker_width=256, T=2 shared applications:
    every source has two edge tiles, every CTA of k_dy / k_dh walks many sources / tiles.  Reference: autograd through
    the mask-consistent forward (fp32 torch ops on the GPU, TF32 off, edge-chunked), node-level ReLUs evaluated at the
    CUDA path's own conv outputs."""
    from graph_pde_b200 import graphs
    from graph_pde_b200.nn_conv import NNConv_old
    s, r, w, kw, T = 85, 0.10, 64, 256, 2
    dev = torch.device(DEV)
    ei = graphs.ball_connectivity(s, r, dev, True)
    _, _, ea = graphs.darcy_sample(s, r, dev, seed=2, edge_index=ei)
    ws, bs, root, bias = O.reference_init(w, w, [6, kw, kw, w * w], seed=0)
    torch.manual_seed(1)
    x0 = torch.randn(s * s, w, device=dev)
    gout = torch.randn(s * s, w, device=dev)
    conv = make_conv(NNConv_old, ws, bs, root, bias, 'mean', w, w, 'f16', dev)
    conv_outs = []
    hook = conv.register_forward_hook(lambda m, i, o: conv_outs.append(o.detach()))
    xd = x0.clone().requires_grad_(True)
    h = xd
    for _ in range(T):
        h = torch.relu(conv(h, ei, ea))
    (h * gout).sum().backward()
    hook.remove()
    lin_d = [m for m in conv.nn.layers if isinstance(m, torch.nn.Linear)]
    got = {'x': xd.grad, 'root': conv.root.grad, 'bias': conv.bias.grad}
    for i, l in enumerate(lin_d):
        got['W%d' % i], got['b%d' % i] = l.weight.grad, l.bias.grad
    got = {k: v.detach().cpu() for k, v in got.items()}
    conv._h_cache.clear()
    conv._tstate = None
    torch.cuda.empty_cache()
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        leaves = [t.to(dev).clone().requires_grad_(True) for t in [x0.cpu()] + ws + bs + [root, bias]]
        xr, wr, br, rr, bbr = leaves[0], leaves[1:4], leaves[4:7], leaves[7], leaves[8]
        hr = xr
        for k in range(T):
            o = emulated_nnconv_forward(hr, ei, ea, wr, br, rr, bbr, 'mean', 'f16', edge_chunk=1 << 17)
            hr = torch.relu(o + (conv_outs[k] - o).detach())
        (hr * gout).sum().backward()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    ref = {'x': xr.grad, 'root': rr.grad, 'bias': bbr.grad}
    for i in range(3):
        ref['W%d' % i], ref['b%d' % i] = wr[i].grad, br[i].grad
    errs = {k: _relerr(got[k], ref[k]) for k in ref}
    print('config-2-size gradient errors vs mask-consistent fp32 autograd:', errs)
    bad = {k: v for k, v in errs.items() if not v < 5e-3}
    assert not bad, (bad, errs)


def test_kept_and_recomputed_hidden_activations_give_the_same_gradients(monkeypatch):
    """Training keeps h_1..h_{L-2} of the forward when they fit NNCONV_B200_KEEP_ACTS_BYTES, else the deferred pass
    recomputes them per batch: same gradients either way (4-layer MLP: two kept layers)."""
    from graph_pde_b200 import nn_conv
    from graph_pde_b200.nn_conv import NNConv_old
    gen = torch.Generator().manual_seed(23)
    N, E, w = 200, 6000, 64
    ei = _graph(gen, N, E, hub=True)
    ea = torch.randn(E, 6, generator=gen)
    x = torch.randn(N, w, generator=gen)
    gout = torch.randn(N, w, generator=gen)
    torch.manual_seed(4)
    mlp = DenseNetLike([6, 128, 64, 192, w * w])
    lin = [m for m in mlp.layers if isinstance(m, torch.nn.Linear)]
    ws, bs = [l.weight.detach().clone() for l in lin], [l.bias.detach().clone() for l in lin]
    grads = []
    root = torch.randn(w, w, generator=gen) * 0.1
    for budget in (64 << 30, 0):
        monkeypatch.setattr(nn_conv, '_KEEP_ACTS_MAX_BYTES', budget)
        conv = make_conv(NNConv_old, ws, bs, root, None, 'mean', w, w, 'f16', DEV)
        xd = x.to(DEV).requires_grad_(True)
        h = torch.relu(conv(xd, ei.to(DEV), ea.to(DEV)))
        kept = conv._tstate.acts is not None
        assert kept == (budget > 0)
        (h * gout.to(DEV)).sum().backward()
        lin_d = [m for m in conv.nn.layers if isinstance(m, torch.nn.Linear)]
        grads.append([xd.grad] + [l.weight.grad for l in lin_d] + [l.bias.grad for l in lin_d])
    for a, b in zip(*grads):
        assert _relerr(a, b) < 1e-5
