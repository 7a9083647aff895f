"""The wgmma GEMM at its widest tiles (N = 1024) with several tiles per CTA and a partial last m-block, so every
ring stage and barrier phase wraps; and the edge-feature pass split into several chunks,
checked row by row at every chunk boundary.  pytest -m gpu."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda:0')
M_TILES = 20000 + 77          # BLOCK_N = 256: 157 m-blocks x 4 n-blocks = 628 tiles, ~4.8 per CTA on 132 SMs
                              # (16 k-blocks each: the 3-stage ring wraps many times); last m-block 109 rows


def _lib():
    from graph_pde_b200 import _lib
    L = _lib.lib()
    _lib.check(L.nnconv_init())
    return _lib, L


def _relerr(out, ref):
    return float((out.double() - ref).abs().max() / ref.abs().max())


def _operands(dt, M, N, K, seed):
    g = torch.Generator(device='cpu').manual_seed(seed)
    A = (torch.randn(M, K, generator=g) * 0.1).to(DEV).to(dt)
    B = (torch.randn(N, K, generator=g) * 0.1).to(DEV).to(dt)
    return g, A, B


@pytest.mark.parametrize('prec,dt', [('f16', torch.float16), ('bf16', torch.bfloat16)])
def test_plain_epilogue_n1024_partial_m(prec, dt):
    _l, L = _lib()
    M, N, K = M_TILES, 1024, 1024
    g, A, B = _operands(dt, M, N, K, 1)
    bias = torch.randn(N, generator=g).to(DEV)
    C = torch.full((M, N), float('nan'), device=DEV, dtype=dt)
    _l.check(L.nnconv_gemm_16b(_l.PREC[prec], ctypes.c_void_p(A.data_ptr()), M, K, ctypes.c_void_p(B.data_ptr()), N,
                               ctypes.c_void_p(bias.data_ptr()), 1, ctypes.c_void_p(C.data_ptr()),
                               ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    ref = torch.relu(A.double() @ B.double().t() + bias.double())
    assert _relerr(C, ref) < (2e-3 if prec == 'f16' else 1.6e-2)


@pytest.mark.parametrize('prec,dt', [('f16', torch.float16), ('bf16', torch.bfloat16)])
def test_mask_and_f32_epilogues_n1024(prec, dt):
    _l, L = _lib()
    M, N, K = M_TILES, 1024, 1024
    g, A, B = _operands(dt, M, N, K, 2)
    act = torch.relu(torch.randn(M, N, generator=g)).to(DEV).to(dt)          # ~half zeros
    st = torch.cuda.current_stream().cuda_stream
    ref = A.double() @ B.double().t()
    C = torch.full((M, N), float('nan'), device=DEV, dtype=dt)
    _l.check(L.nnconv_gemm_16b_ex(_l.PREC[prec], A.data_ptr(), M, K, B.data_ptr(), N, None, 0, C.data_ptr(), N,
                                  act.data_ptr(), N, 0, st))
    torch.cuda.synchronize()
    keep = act > 0
    assert bool((C[~keep] == 0).all())
    assert _relerr(C, ref * keep) < (4e-3 if prec == 'f16' else 3e-2)
    C32 = torch.full((M, N), float('nan'), device=DEV)
    _l.check(L.nnconv_gemm_16b_ex(_l.PREC[prec], A.data_ptr(), M, K, B.data_ptr(), N, None, 0, C32.data_ptr(), N, None,
                                  0, 1, st))
    torch.cuda.synchronize()
    assert _relerr(C32, ref) < 1e-4


def _edge_case(n_nodes=3000, E=20037, w=16, kw=1024, seed=0):
    """A graph grouped by source (the plan keeps the caller's edge order) and a [6, kw, kw, w*w] edge MLP."""
    from graph_pde_b200.nn_conv import NNConv_old
    g = torch.Generator(device='cpu').manual_seed(seed)
    src = torch.sort(torch.randint(0, n_nodes, (E,), generator=g)).values
    dst = torch.randint(0, n_nodes, (E,), generator=g)
    ei = torch.stack([src, dst]).to(DEV)
    ea = torch.rand(E, 6, generator=g).to(DEV)
    torch.manual_seed(seed)
    mlp = torch.nn.Sequential(torch.nn.Linear(6, kw), torch.nn.ReLU(), torch.nn.Linear(kw, kw), torch.nn.ReLU(),
                              torch.nn.Linear(kw, w * w))
    conv = NNConv_old(w, w, mlp, aggr='mean', precision='f16').to(DEV)
    return conv, mlp, ei, ea, n_nodes


def _edge_features(conv, ei, ea, n_nodes, ws_bytes, monkeypatch):
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_EF_WS_BYTES', ws_bytes)
    plan = nn_conv.get_plan(ei, n_nodes)
    prepared = conv._get_prepared('f16')
    conv._h_cache.clear()
    n0 = nn_conv.stats['launches']
    h = conv.edge_features(plan, prepared, ea)
    torch.cuda.synchronize()
    return h, nn_conv.stats['launches'] - n0


def test_edge_features_across_chunks(monkeypatch):
    conv, mlp, ei, ea, n_nodes = _edge_case()
    E, kw = ea.size(0), 1024
    E_pad = (E + 127) // 128 * 128
    h, launches = _edge_features(conv, ei, ea, n_nodes, 16 << 20, monkeypatch)
    assert launches >= 3 * 3, launches             # per chunk: a1 build + first Linear, hidden Linear
    # chunk-major [kw / 64][E_pad][64] -> [E_pad, kw]
    hh = h.view(torch.float16)[:kw * E_pad].view(kw // 64, E_pad, 64).permute(1, 0, 2).reshape(E_pad, kw)
    with torch.no_grad():
        l1, l2 = mlp[0], mlp[2]
        h1 = torch.relu(ea.double() @ l1.weight.double().t() + l1.bias.double())
        ref = torch.relu(h1 @ l2.weight.double().t() + l2.bias.double())
    got = hh[:E].double()
    scale = float(ref.abs().max())
    err_rows = (got - ref).abs().max(dim=1).values / scale
    assert float(err_rows.max()) < 4e-3
    # chunks (and m-blocks) start at multiples of 128 rows: both rows around every such boundary
    for r in [b + d for b in range(128, E, 128) for d in (-1, 0)] + [E - 1]:
        assert float(err_rows[r]) < 4e-3, r
    assert bool(torch.isfinite(hh[E:E_pad].float()).all())
    # splitting the pass into chunks does not change a single bit
    h_one, launches1 = _edge_features(conv, ei, ea, n_nodes, 2 << 30, monkeypatch)
    assert launches1 == 3
    hh1 = h_one.view(torch.float16)[:kw * E_pad].view(kw // 64, E_pad, 64).permute(1, 0, 2).reshape(E_pad, kw)
    assert torch.equal(hh1[:E], hh[:E])


def test_overflow_in_last_partial_tile_is_reported(monkeypatch):
    conv, mlp, ei, ea, n_nodes = _edge_case(E=1000 + 3)
    with torch.no_grad():
        mlp[2].weight.mul_(200.0)                   # hidden activations ~1e2 for edge attributes in [0, 1)
    _edge_features(conv, ei, ea, n_nodes, 2 << 30, monkeypatch)          # in range: no report
    ea = ea.clone()
    ea[-1] = 1.0e3                                  # the last edge only (row 1002, 8th and partial m-block): ~1e5
    with pytest.raises(FloatingPointError):
        _edge_features(conv, ei, ea, n_nodes, 2 << 30, monkeypatch)
