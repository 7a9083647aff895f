"""Every forward path on exact integer probes (tests/probes.py): with aggr='add' the library must equal the fp64
reference bit for bit at every node, so one lost, doubled or misrouted edge fails at the node it touches, and the
schedules (fused, per-batch, streamed, formulation B, graph replay) agree bitwise.  aggr='mean' is compared node by
node against a bound derived from each node's degree that is smaller than the node's smallest message."""
import ctypes

import pytest
import torch

from oracle import nnconv_oracle as O
from tests import probes as P
from tests.helpers import oracle_stack_on_cuda

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


@pytest.fixture(autouse=True)
def formulation_c(monkeypatch):
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_EDGE_KERNELS', 'off')


def _cls():
    from graph_pde_b200.nn_conv import NNConv_old
    return NNConv_old


_REF = {}


def _reference(p, aggr, x=None, key=None):
    """fp64 oracle on the CPU: (out, messages [E, cout] in the caller's edge order)."""
    if key is not None and key in _REF:
        return _REF[key]
    src, dst = (t.cpu() for t in p.src_dst())
    x = p.x[0] if x is None else x
    ea = p.ea.double().cpu()
    k = O.dense_net(ea, p.ws, p.bs).view(-1, p.cin, p.cout)
    msg = torch.bmm(x[src].unsqueeze(1), k).squeeze(1)
    out = O.nnconv_forward(x, torch.stack([src, dst]), ea, p.ws, p.bs, p.root, p.bias, aggr)
    if key is not None:
        _REF[key] = (out, msg)
    return out, msg


def assert_matches(out, p, aggr, ref, msg, x=None):
    """add: bitwise at every node.  mean: |out - ref| within (deg + 2) 2^-24 of the node's sum of |terms| per channel
    (deg fp32 adds, and the rounding of inv_deg and of each m * inv_deg),
    a bound the reference first shows to be smaller than the node's smallest message (channel 0 of every message is
    x_src[0] >= 1), so one edge lost, doubled or misrouted still fails."""
    out = out.detach().double().cpu()
    if aggr == 'add':
        bad = (out != ref).any(1)
        assert not bool(bad.any()), ('nodes differ', torch.nonzero(bad).flatten()[:20].tolist(),
                                     float((out - ref).abs().max()))
        return
    bound, smallest, has_in = _mean_bound(p, msg, p.x[0] if x is None else x)
    assert bool((bound[has_in, 0] < smallest[has_in]).all()), 'the mean bound would absorb one message'
    err = (out - ref).abs()
    bad = (err > bound).any(1)
    assert not bool(bad.any()), ('nodes beyond the bound', torch.nonzero(bad).flatten()[:20].tolist())


def _mean_bound(p, msg, x):
    """Per node and channel bound of aggr='mean', each node's smallest channel-0 message / deg, nodes with in-edges."""
    src, dst = (t.cpu() for t in p.src_dst())
    N = p.n_nodes
    deg = torch.zeros(N, dtype=torch.float64).index_add_(0, dst, torch.ones(dst.numel(), dtype=torch.float64))
    init = torch.zeros(N, p.cout, dtype=torch.float64)
    if p.root is not None:
        init = init + (x.abs() @ p.root.abs())
    if p.bias is not None:
        init = init + p.bias.abs()
    inv = 1.0 / deg.clamp(min=1)
    s = init.index_add(0, dst, msg.abs() * inv[dst].unsqueeze(1))
    bound = (deg + 2).unsqueeze(1) * 2.0 ** -24 * s
    smallest = torch.full((N,), float('inf'), dtype=torch.float64).scatter_reduce(
        0, dst, msg[:, 0].abs() * inv[dst], 'amin')
    return bound, smallest, deg > 0


def _run(p, precision, aggr, **kw):
    conv = p.conv(_cls(), precision, aggr, DEV, **kw)
    with torch.no_grad():
        return conv(p.x[0].float().to(DEV), p.ei.to(DEV), p.ea.to(DEV)), conv


# ---- 0. the tensor cores sum integers exactly within the budget --------------------------------------------------------
@pytest.mark.parametrize('prec,dt,lim', [('f16', torch.float16, 64), ('bf16', torch.bfloat16, 64)])
def test_tensor_core_sums_at_the_budget_limit_are_exact(prec, dt, lim):
    """nnconv_gemm_16b_ex (fp32 out) and nnconv_gemm_tn_16b on integer operands whose sums of |terms| reach 2^22
    (K = 1024 terms of 64 * 64; R = 1024 rows of 64 * 64 for gemm_tn, split over rows and added with fp32 atomics)
    equal an int64 matmul: the budget of tests/probes.py holds on this hardware."""
    from graph_pde_b200 import _lib
    L = _lib.lib()
    _lib.check(L.nnconv_init())
    g = torch.Generator().manual_seed(5)
    M, K, N = 512, 1024, 256
    A = torch.randint(-lim, lim + 1, (M, K), generator=g)
    B = torch.randint(-lim, lim + 1, (N, K), generator=g)
    A[0], B[0] = lim, lim                                   # C[0, 0] = 2^22 exactly
    A[1], B[1] = lim, -lim
    # C[2, 2]: a same-sign run of 64 * 64 products up to 2^22 - 2^13, then unit products: running sums near 2^22
    # must keep every later +-1 exactly
    A[2, :1022], B[2, :1022] = lim, lim
    A[2, 1022:], B[2, 1022:] = torch.tensor([1, -1]), torch.tensor([1, 1])
    A[3, :1022], B[3, :1022] = lim, lim                     # C[3, 3] = 2^22 - 2^13 + 1 + 1
    A[3, 1022:], B[3, 1022:] = 1, 1
    ref = A @ B.t()
    assert int(ref[0, 0]) == 1 << 22 and int(ref[3, 3]) == (1 << 22) - (1 << 13) + 2
    Ad, Bd = A.to(DEV, dt), B.to(DEV, dt)
    C = torch.zeros(M, N, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(L.nnconv_gemm_16b_ex(_lib.PREC[prec], Ad.data_ptr(), M, K, Bd.data_ptr(), N, None, 0, C.data_ptr(), N,
                                    None, 0, 1, st))
    torch.cuda.synchronize()
    assert torch.equal(C.cpu().to(torch.int64), ref)
    R, M2, N2 = 1024, 128, 64
    lda = M2 + 64                                           # A as the backward lays it out: wider than the M it reads
    A2 = torch.randint(-lim, lim + 1, (R, lda), generator=g)
    B2 = torch.randint(-lim, lim + 1, (R, N2), generator=g)
    A2[:, 0], B2[:, 0] = lim, lim
    A2[:-2, 1], B2[:-2, 1] = lim, lim                       # C2[1, 1]: a run to 2^22 - 2^13, then +-1 products
    A2[-2:, 1], B2[-2:, 1] = torch.tensor([1, 1]), torch.tensor([1, -1])
    C2 = torch.zeros(M2, N2, device=DEV)
    A2d, B2d = A2.to(DEV, dt), B2.to(DEV, dt)
    _lib.check(L.nnconv_gemm_tn_16b(_lib.PREC[prec], A2d.data_ptr(), lda, B2d.data_ptr(), N2, R, M2, N2, C2.data_ptr(), N2,
                                    1.0, st))
    torch.cuda.synchronize()
    ref2 = A2[:, :M2].t() @ B2
    assert int(ref2[0, 0]) == 1 << 22
    assert torch.equal(C2.cpu().to(torch.int64), ref2)


# ---- 1. every application path ----------------------------------------------------------------------------------------
# path name: (library options, nn_conv module settings)
PATHS = {
    'fused_coop': ({}, {}),
    'fused_no_coop': ({'no_coop': 1}, {}),
    'per_batch_pdl': ({'no_fuse': 1}, {}),
    'per_batch_stream_order': ({'no_fuse': 1, 'no_pipe': 1}, {}),
    'scatter_mode0': ({'scatter_mode': 0}, {}),
    'gemm_direct_store': ({'gemm_direct_store': 1}, {}),
    'apply_passes2': ({'apply_passes': 2}, {}),
    'many_flag_batches': ({}, {'_Y_BYTES': 3 * 4 * 64 * 128 * 2}),
}
SPLIT_PATHS = ('fused_coop', 'fused_no_coop', 'scatter_mode0', 'many_flag_batches')   # f16x2 has no per-batch schedule


@pytest.mark.parametrize('aggr', ['add', 'mean'])
@pytest.mark.parametrize('path', list(PATHS))
@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2'])
def test_application_paths(precision, path, aggr, lib_options, monkeypatch):
    if precision == 'f16x2' and path not in SPLIT_PATHS:
        pytest.skip('f16x2 runs the fused kernel only')
    from graph_pde_b200 import nn_conv
    opts, mods = PATHS[path]
    for k, v in opts.items():
        lib_options(k, v)
    for k, v in mods.items():
        monkeypatch.setattr(nn_conv, k, v * (2 if precision == 'f16x2' else 1))
    p = P.probe(P.FORWARD, 'mixed', precision=precision)
    ref, msg = _reference(p, aggr, key=('mixed', aggr, bool(P.wide_options(P.FORWARD, 'mixed', precision))))
    out, _ = _run(p, precision, aggr)
    assert_matches(out, p, aggr, ref, msg)


@pytest.mark.parametrize('name', ['mixed_wide_ea', 'partial_tiles', 'hub_batches', 'asymmetric_t2s', 'batch'])
@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2'])
def test_graphs(precision, name, monkeypatch):
    """Partial last tiles of every box height, a hub across ~100 flag batches, flow target_to_source on a graph with
    no reverse edges, a block-diagonal batch, and edge attributes whose first-layer split has non-zero lo halves."""
    from graph_pde_b200 import nn_conv
    if name == 'hub_batches':
        monkeypatch.setattr(nn_conv, '_Y_BYTES', 3 * 4 * 64 * 256 * 2 * (2 if precision == 'f16x2' else 1))
    p = P.probe(P.FORWARD, name, precision=precision)
    for aggr in ('add', 'mean'):
        ref, msg = _reference(p, aggr)
        out, _ = _run(p, precision, aggr)
        assert_matches(out, p, aggr, ref, msg)


@pytest.mark.parametrize('name,precision', [(n, pr) for n in ('nc16', 'nc32', 'nc48', 'out80', 'out96', 'out112', 'out128',
                                                               'kp1088', 'kin24_2layer', 'kin24_3layer', 'single_linear',
                                                               'fp32_out40') for pr in P.FORWARD[n][-1]])
def test_shapes(name, precision, monkeypatch):
    """Fused out in {16, 32, 48}, per-batch out in {80, 96, 112, 128}, Kp = 1088 (17 passes), the CUDA-core first
    layer (k_in > 20) into h and into the ping-pong buffer, the identity first layer, and precision fp32."""
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_EF_WS_BYTES', 1 << 20)
    p = P.probe(P.FORWARD, name, precision=precision)
    ref, msg = _reference(p, 'add')
    out, _ = _run(p, precision, 'add')
    assert_matches(out, p, 'add', ref, msg)


def _h_bytes(conv, p):
    from graph_pde_b200 import _lib, nn_conv
    plan = nn_conv.get_plan(p.ei.to(DEV), p.n_nodes, conv.flow)
    prep = conv._get_prepared(conv.precision)
    h_b, ws_b = ctypes.c_size_t(), ctypes.c_size_t()
    _lib.check(_lib.lib().nnconv_edge_features_sizes(plan.handle, prep.handle, 1 << 20, ctypes.byref(h_b),
                                                     ctypes.byref(ws_b)))
    return h_b.value


@pytest.mark.parametrize('chunk_bytes', [3 << 20, 300007])
@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2'])
def test_streamed_edge_features(precision, chunk_bytes, monkeypatch):
    """Budget 0, half of h, and a prefix that ends inside the hub source's units; chunks that end inside the hub:
    bitwise equal to the reference and to the cached run."""
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_EF_WS_BYTES', chunk_bytes)
    p = P.probe(P.FORWARD, 'mixed', precision=precision)
    ref, msg = _reference(p, 'add', key=('mixed', 'add', bool(P.wide_options(P.FORWARD, 'mixed', precision))))
    cached, conv = _run(p, precision, 'add')
    assert_matches(cached, p, 'add', ref, msg)
    hb = _h_bytes(conv, p)
    src = p.src_dst()[0].cpu()
    counts = torch.bincount(src, minlength=p.n_nodes)
    hub = int(counts.argmax())
    g_hub, deg_hub = int(counts[:hub].sum()), int(counts[hub])
    row = hb // ((p.ei.size(1) + 127) // 128 * 128)          # h bytes per edge row
    straddle = (g_hub + deg_hub - 1) * row                    # E_res: a unit boundary inside the hub
    for budget in (0, hb // 2, straddle):
        c0 = nn_conv.stats['streamed_chunk_passes']
        out, conv = _run(p, precision, 'add', edge_feature_bytes=budget)
        assert nn_conv.stats['streamed_chunk_passes'] > c0
        if budget == straddle:                  # the prefix ends inside the hub source's units
            e_res = next(iter(conv._h_cache.values())).E_res
            assert g_hub < e_res < g_hub + deg_hub, (g_hub, deg_hub, e_res)
        assert torch.equal(out, cached), budget
        assert_matches(out, p, 'add', ref, msg)


@pytest.mark.parametrize('name', ['edge_v64_src', 'edge_v64', 'edge_v32', 'edge_scalar_src', 'edge_scalar'])
@pytest.mark.parametrize('precision', ['f16', 'bf16'])
def test_formulation_b(precision, name, monkeypatch):
    """Per-edge kernel matrices: k_apply_edge_src_v / k_apply_edge_v at 64x64 and 32x32, the scalar kernels otherwise;
    plain applications and residual steps."""
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_EDGE_KERNELS', 'on')
    p = P.probe(P.FORWARD, name)
    n0 = nn_conv.stats['edge_kernel_passes']
    for aggr in ('add', 'mean'):
        ref, msg = _reference(p, aggr)
        out, conv = _run(p, precision, aggr)
        assert_matches(out, p, aggr, ref, msg)
    assert nn_conv.stats['edge_kernel_passes'] > n0
    if p.cin == p.cout:
        _residual(p, precision)


def _residual(p, precision):
    xr = torch.relu(p.x[0])
    ref, _ = _reference(p, 'add', x=xr)
    conv = p.conv(_cls(), precision, 'add', DEV)
    with torch.no_grad():
        z = conv.residual_step(p.x[0].float().to(DEV), p.ei.to(DEV), p.ea.to(DEV), relu_in=True)
    assert torch.equal(z.double().cpu(), xr + ref)


@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2'])
def test_residual_step(precision):
    """residual_step (RELU_IN | RESIDUAL folded into the node prep) on formulation C."""
    _residual(P.probe(P.FORWARD, 'mixed'), precision)


@pytest.mark.parametrize('precision', ['f16', 'f16x2'])
def test_graphed_forward_replay(precision):
    """A captured forward replays to the eager output bitwise."""
    from graph_pde_b200.capture import GraphedForward
    p = P.probe(P.FORWARD, 'mixed')
    conv = p.conv(_cls(), precision, 'add', DEV)
    x, ei, ea = p.x[0].float().to(DEV), p.ei.to(DEV), p.ea.to(DEV)
    with torch.no_grad():
        eager = conv(x, ei, ea)
    gf = GraphedForward(lambda xx: conv(xx, ei, ea), x)
    out = gf.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
    ref, msg = _reference(p, 'add', key=('mixed', 'add'))
    assert_matches(out, p, 'add', ref, msg)


# ---- 2. one edge changed: the probe detects it where it happened -------------------------------------------------------
@pytest.mark.parametrize('change', ['delete', 'duplicate', 'redirect'])
@pytest.mark.parametrize('aggr', ['add', 'mean'])
def test_one_changed_edge_fails_exactly_where_it_lands(change, aggr):
    """The library on a copy of the graph with one edge deleted, duplicated or sent to another target, against the
    reference of the unmodified graph: the mismatch is at exactly the nodes the change touched."""
    p = P.probe(P.FORWARD, 'mixed')
    ref, msg = _reference(p, aggr, key=('mixed', aggr))
    ei = p.ei.clone()
    ea = p.ea.clone()
    e = 1234
    s, d = int(ei[0, e]), int(ei[1, e])
    if change == 'delete':
        keep = torch.arange(ei.size(1)) != e
        ei, ea, touched = ei[:, keep], ea[keep], {d}
    elif change == 'duplicate':
        ei, ea, touched = torch.cat([ei, ei[:, e:e + 1]], 1), torch.cat([ea, ea[e:e + 1]]), {d}
    else:
        d2 = (d + 17) % p.n_nodes
        ei[1, e] = d2
        touched = {d, d2}
    conv = p.conv(_cls(), 'f16', aggr, DEV)
    with torch.no_grad():
        out = conv(p.x[0].float().to(DEV), ei.to(DEV), ea.to(DEV))
    with pytest.raises(AssertionError) as err:
        assert_matches(out, p, aggr, ref, msg)
    assert 'nodes' in str(err.value)
    out = out.double().cpu()
    if aggr == 'add':
        bad = (out != ref).any(1)
    else:
        bad = ((out - ref).abs() > _mean_bound(p, msg, p.x[0])[0]).any(1)
    assert set(torch.nonzero(bad).flatten().tolist()) == touched, (torch.nonzero(bad).flatten().tolist(), touched)


# ---- 3. full scale: KernelNN's edge network on the 241^2 mesh -----------------------------------------------------------
@pytest.mark.parametrize('precision,budget', [('f16', None), ('f16', 24 << 30), ('f16x2', 'auto')])
def test_darcy241_one_application(precision, budget):
    """One application at 241^2 (58,081 nodes, 24,557,297 edges, ~423 in-edges per node), bitwise at every node
    against the oracle's torch ops on the GPU (fp32, TF32 off: exact on the probe): the whole h cached, a 24 GB budget,
    and f16x2 with the budget from the free memory (streamed)."""
    import gc
    from graph_pde_b200 import nn_conv
    nn_conv.clear_caches()          # the plans of the other 241^2 cases
    gc.collect()
    p = P.probe(P.FORWARD, 'darcy241', DEV)
    kw = {} if budget in (None, 'auto') else {'edge_feature_bytes': budget}
    conv = p.conv(_cls(), precision, 'add', DEV, **kw)
    x, ei, ea = p.x[0].float().to(DEV), p.ei, p.ea
    c0 = nn_conv.stats['streamed_chunk_passes']
    failure = None
    fragments = None
    if budget == 'auto':
        # 1.5 GiB of the caching allocator's 2 MiB segments left three-quarters free: memory it holds but cannot hand
        # to the 2 GiB workspaces the automatic budget must leave room for
        blocks = [torch.empty(512 << 10, dtype=torch.uint8, device=DEV) for _ in range(4096)]
        fragments = blocks[::4]
        del blocks
    try:
        with torch.no_grad():
            out = conv(x, ei, ea)
    except torch.cuda.OutOfMemoryError as e:
        failure = str(e)            # not re-raised: its traceback would keep the edge features alive for later tests
    del fragments
    if failure is not None:
        conv.invalidate()
        pytest.fail(failure)
    streamed = nn_conv.stats['streamed_chunk_passes'] > c0
    assert streamed == (budget is not None)
    out = out.cpu()
    conv.invalidate()
    del conv
    torch.cuda.empty_cache()
    ws = [w.float().to(DEV) for w in p.ws]
    bs = [b.float().to(DEV) for b in p.bs]
    ref = oracle_stack_on_cuda(x, ei, ea, ws, bs, p.root.float().to(DEV), p.bias.float().to(DEV), 1, aggr='add',
                               edge_chunk=1 << 17, relu_last=False)[0].cpu()
    bad = (out != ref).any(1)
    assert not bool(bad.any()), ('nodes differ', int(bad.sum()), torch.nonzero(bad).flatten()[:20].tolist())
