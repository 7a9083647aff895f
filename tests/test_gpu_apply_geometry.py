"""Geometry of the persistent application kernel (k_apply_tc): the default Y ring is sized from the device's L2, and
schedules with many small source batches, hub sources and partial tiles of every TMA box height give the oracle's
answer in every 16-bit precision."""
import ctypes
import math

import pytest
import torch

from oracle import nnconv_oracle as O
from tests.helpers import TOL, DenseNetLike, make_conv, rel_err

pytestmark = pytest.mark.gpu

MAX_PIPE_BATCHES = 1 << 14      # flag table of one application (api.cu: kMaxPipeBatches)


@pytest.fixture(scope='module')
def dev():
    assert torch.cuda.is_available()
    return torch.device('cuda:0')


@pytest.fixture(autouse=True)
def formulation_c(monkeypatch):
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_EDGE_KERNELS', 'off')


def _cls():
    from graph_pde_b200.nn_conv import NNConv_old
    return NNConv_old


def _params(layers, w, seed=3):
    torch.manual_seed(seed)
    mlp = DenseNetLike(layers)
    lin = [m for m in mlp.layers if isinstance(m, torch.nn.Linear)]
    return ([l.weight.detach() for l in lin], [l.bias.detach() for l in lin], torch.randn(w, w) * 0.1,
            torch.randn(w) * 0.1)


def _ring_option():
    from graph_pde_b200 import _lib
    v = ctypes.c_int()
    _lib.check(_lib.lib().nnconv_get_option(b'ring', ctypes.byref(v)))
    return v.value


@pytest.mark.parametrize('s,r', [(241, 0.05), (85, 0.10)])
def test_default_y_ring_fits_the_l2(dev, s, r):
    """nnconv_apply_sizes(want_y_bytes = 0) sizes the Y ring from the L2 the device reports: the ring fits it, every
    slot holds at least one 128-source m-block of the Y GEMM (or every source), and the batches of the graph stay
    within the flag table of one application."""
    from graph_pde_b200 import _lib, graphs, nn_conv
    w, kw = 64, 1024
    ws, bs, root, bias = _params([6, 64, kw, w * w], w)
    conv = make_conv(_cls(), ws, bs, root, bias, 'mean', w, w, 'f16', dev)
    ei = graphs.ball_connectivity(s, r, dev, True)
    plan = nn_conv.get_plan(ei, s * s, conv.flow)
    prep = conv._get_prepared('f16')
    L = _lib.lib()
    per_node = w * kw * 2                        # one source's Y matrix, [out, Kp] fp16
    ws_default, ws_one = ctypes.c_size_t(), ctypes.c_size_t()
    _lib.check(L.nnconv_apply_sizes(plan.handle, prep.handle, 0, ctypes.byref(ws_default)))
    _lib.check(L.nnconv_apply_sizes(plan.handle, prep.handle, per_node, ctypes.byref(ws_one)))
    nodes = (ws_default.value - ws_one.value) // per_node + 1
    l2 = torch.cuda.get_device_properties(dev).L2_cache_size
    assert 0 < nodes * per_node <= l2, (nodes, l2)
    ring = _ring_option()
    nb = min(nodes // ring, plan.n_src)
    if nb >= 128:
        nb = nb // 128 * 128
    assert nb >= min(128, plan.n_src) or nodes == plan.n_src, (nodes, ring, nb)
    assert math.ceil(plan.n_src / nb) <= MAX_PIPE_BATCHES
    # the smallest default batch (one m-block per slot) keeps meshes of up to 2M sources within the flag table
    assert math.ceil(2_000_000 / 128) <= MAX_PIPE_BATCHES


def _graph_with_degrees(degrees, N, dev, seed):
    gen = torch.Generator().manual_seed(seed)
    src = torch.cat([torch.full((d,), i, dtype=torch.int64) for i, d in enumerate(degrees)])
    dst = torch.randint(0, N, (src.numel(),), generator=gen)
    perm = torch.randperm(src.numel(), generator=gen)     # unsorted edge order
    ei = torch.stack([src[perm], dst[perm]])
    ea = torch.randn(src.numel(), 6, generator=gen)
    return ei.to(dev), ea.to(dev)


def _check(dev, ei, ea, N, prec, layers, w, seed):
    ws, bs, root, bias = _params(layers, w, seed)
    conv = make_conv(_cls(), ws, bs, root, bias, 'mean', w, w, prec, dev)
    gen = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(N, w, generator=gen)
    with torch.no_grad():
        out = conv(x.to(dev), ei, ea)
    ref = O.nnconv_forward(x.double(), ei.cpu(), ea.double().cpu(), [v.double() for v in ws], [v.double() for v in bs],
                           root.double(), bias.double(), aggr='mean')
    return rel_err(out, ref)


@pytest.mark.parametrize('prec', ['f16', 'bf16', 'f16x2'])
def test_hub_source_across_many_small_batches(dev, prec, monkeypatch):
    """A hub source with 2,500 out-edges (10 two-tile units) among ~380 ordinary sources, with a Y ring of 3 x 4
    sources: about 100 batches go through the okY / okC flags while the hub's units are still streaming."""
    from graph_pde_b200 import nn_conv
    w, kw = 64, 256
    N, E = 400, 6000
    gen = torch.Generator().manual_seed(17)
    src = torch.randint(0, N - 20, (E,), generator=gen)
    dst = torch.randint(0, N, (E,), generator=gen)
    src[:2500] = 200                              # the hub sits in the middle of the source order
    ei = torch.stack([src, dst]).to(dev)
    ea = torch.randn(E, 6, generator=gen).to(dev)
    per_node = w * kw * 2 * (2 if prec == 'f16x2' else 1)
    monkeypatch.setattr(nn_conv, '_Y_BYTES', 3 * 4 * per_node)
    err = _check(dev, ei, ea, N, prec, [6, 64, kw, w * w], w, seed=5)
    assert err < TOL[prec], (prec, err)


@pytest.mark.parametrize('prec', ['f16', 'bf16', 'f16x2'])
def test_partial_last_tile_of_every_box_height(dev, prec):
    """Out-degrees whose last 128-edge tile holds 1..128 rows, so that every one of the 8 A-tile box heights
    (16 * ceil(rows / 16)) is a partial last tile somewhere, plus one- and two-tile units."""
    w, kw = 64, 128
    degrees = [1, 15, 16, 17, 31, 33, 48, 50, 64, 65, 80, 90, 97, 100, 113, 120, 127, 128, 129, 200, 255, 256, 257, 300,
               383, 384, 385, 511]
    N = 600
    ei, ea = _graph_with_degrees(degrees, N, dev, seed=9)
    err = _check(dev, ei, ea, N, prec, [6, 32, kw, w * w], w, seed=8)
    assert err < TOL[prec], (prec, err)
