"""The forward epilogue of the wgmma GEMM (bias, ReLU and the 16-bit rounding on the accumulator fragments, stmatrix
into the swizzled staging) at every tile width, at M around the 128-row m-block and at partial last m-blocks, on
both store paths; and the edge-feature pass it writes (chunk-major output, the f16x2 [hi | lo] pairs, the fp16
range check).  pytest -m gpu."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda:0')


def _lib():
    from graph_pde_b200 import _lib
    L = _lib.lib()
    _lib.check(L.nnconv_init())
    return _lib, L


def _operands(dt, M, N, K, seed):
    g = torch.Generator(device='cpu').manual_seed(seed)
    A = (torch.randn(M, K, generator=g) * 0.1).to(DEV).to(dt)
    B = (torch.randn(N, K, generator=g) * 0.1).to(DEV).to(dt)
    bias = torch.randn(N, generator=g).to(DEV)
    return A, B, bias


def _gemm(prec, A, B, bias, relu, M=None):
    _l, L = _lib()
    M = A.size(0) if M is None else M
    N, K = B.shape
    C = torch.full((M, N), float('nan'), device=DEV, dtype=A.dtype)
    _l.check(L.nnconv_gemm_16b(_l.PREC[prec], ctypes.c_void_p(A.data_ptr()), M, K, ctypes.c_void_p(B.data_ptr()), N,
                               ctypes.c_void_p(bias.data_ptr() if bias is not None else 0), relu,
                               ctypes.c_void_p(C.data_ptr()), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    return C


def _check(C, A, B, bias, relu, tol):
    ref = A.double() @ B.double().t()
    if bias is not None:
        ref = ref + bias.double()
    if relu:
        ref = torch.relu(ref)
    assert bool(torch.isfinite(C).all())
    assert float((C.double() - ref).abs().max() / ref.abs().max()) < tol


@pytest.mark.parametrize('M', [1, 127, 128, 129, 255, 20077])
@pytest.mark.parametrize('N', [64, 128, 256, 1024, 4096])
def test_f16_bias_relu(M, N):
    A, B, bias = _operands(torch.float16, M, N, 1024, M + N)
    _check(_gemm('f16', A, B, bias, 1), A, B, bias, 1, 2e-3)


@pytest.mark.parametrize('K', [64, 1024])
@pytest.mark.parametrize('N', [192, 320, 1024])
@pytest.mark.parametrize('prec,dt,tol', [('f16', torch.float16, 2e-3), ('bf16', torch.bfloat16, 1.6e-2)])
def test_no_bias_no_relu_and_partial_n(prec, dt, tol, N, K):
    # N not a multiple of the tile width: the last n-block has columns past N (their pieces are skipped)
    A, B, _ = _operands(dt, 1000, N, K, 7)
    _check(_gemm(prec, A, B, None, 0), A, B, None, 0, tol)


@pytest.mark.parametrize('prec,dt', [('f16', torch.float16), ('bf16', torch.bfloat16)])
@pytest.mark.parametrize('k', [0, 1, 4])
def test_rows_do_not_depend_on_m(prec, dt, k):
    # a launch over the first 128 (2k + 1) rows (an odd m-block count, the last m-block full) gives the same bits for
    # those rows as a launch over all rows
    M = 128 * (2 * k + 1)
    A, B, bias = _operands(dt, M + 300, 1024, 1024, 11)
    full = _gemm(prec, A, B, bias, 1)
    part = _gemm(prec, A, B, bias, 1, M=M)
    assert torch.equal(part, full[:M])


@pytest.mark.parametrize('prec,dt', [('f16', torch.float16), ('bf16', torch.bfloat16)])
def test_direct_store_same_bits(prec, dt):
    from graph_pde_b200 import _lib as lb
    A, B, bias = _operands(dt, 20077, 1024, 1024, 3)
    tma = _gemm(prec, A, B, bias, 1)
    old = lb.get_option('gemm_direct_store')
    lb.set_option('gemm_direct_store', 1)
    try:
        direct = _gemm(prec, A, B, bias, 1)
    finally:
        lb.set_option('gemm_direct_store', old)
    assert torch.equal(direct, tma)


def _edge_case(E, prec, kw=1024, w=16, n_nodes=3000, seed=0):
    from graph_pde_b200.nn_conv import NNConv_old
    g = torch.Generator(device='cpu').manual_seed(seed)
    src = torch.sort(torch.randint(0, n_nodes, (E,), generator=g)).values
    dst = torch.randint(0, n_nodes, (E,), generator=g)
    ei = torch.stack([src, dst]).to(DEV)
    ea = torch.rand(E, 6, generator=g).to(DEV)
    torch.manual_seed(seed)
    mlp = torch.nn.Sequential(torch.nn.Linear(6, kw), torch.nn.ReLU(), torch.nn.Linear(kw, kw), torch.nn.ReLU(),
                              torch.nn.Linear(kw, w * w))
    conv = NNConv_old(w, w, mlp, aggr='mean', precision=prec).to(DEV)
    return conv, mlp, ei, ea, n_nodes


def _edge_features(conv, prec, ei, ea, n_nodes, ws_bytes, monkeypatch):
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_EF_WS_BYTES', ws_bytes)
    plan = nn_conv.get_plan(ei, n_nodes)
    prepared = conv._get_prepared(prec)
    conv._h_cache.clear()
    h = conv.edge_features(plan, prepared, ea)
    torch.cuda.synchronize()
    return h


@pytest.mark.parametrize('ws', [16 << 20, 2 << 30])
def test_f16x2_edge_features_hi_lo(monkeypatch, ws):
    # the [hi | lo] split output of both MLP layers (chunk-major, two chunks at 16 MB of workspace): hi + lo carries the
    # hidden activation far beyond fp16 (whose bound here is 2e-3)
    kw, E = 1024, 3000 + 5
    conv, mlp, ei, ea, n_nodes = _edge_case(E, 'f16x2', kw=kw)
    h = _edge_features(conv, 'f16x2', ei, ea, n_nodes, ws, monkeypatch)
    E_pad = (E + 127) // 128 * 128
    hh = h.view(torch.float16)[:2 * kw * E_pad].view(2 * kw // 64, E_pad, 64).permute(1, 0, 2).reshape(E_pad, 2 * kw)
    val = hh[:E, :kw].double() + hh[:E, kw:].double()
    with torch.no_grad():
        l1, l2 = mlp[0], mlp[2]
        h1 = torch.relu(ea.double() @ l1.weight.double().t() + l1.bias.double())
        ref = torch.relu(h1 @ l2.weight.double().t() + l2.bias.double())
    assert float((val - ref).abs().max() / ref.abs().max()) < 1e-4
    # the lo half is what hi leaves over: no larger than half an fp16 ulp of hi
    hi = hh[:E, :kw].float()
    assert bool((hh[:E, kw:].float().abs() <= torch.clamp(hi.abs(), min=6.1e-5) * 2.0 ** -10).all())


def test_overflow_in_odd_last_m_block_is_reported(monkeypatch):
    # nine m-blocks (the last one of 5 rows): an fp16 overflow in its last row alone is reported
    E = 128 * 8 + 5
    conv, mlp, ei, ea, n_nodes = _edge_case(E, 'f16')
    with torch.no_grad():
        mlp[2].weight.mul_(200.0)
    _edge_features(conv, 'f16', ei, ea, n_nodes, 2 << 30, monkeypatch)
    ea = ea.clone()
    ea[-1] = 1.0e3
    with pytest.raises(FloatingPointError):
        _edge_features(conv, 'f16', ei, ea, n_nodes, 2 << 30, monkeypatch)
