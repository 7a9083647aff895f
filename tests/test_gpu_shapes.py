"""GPU: the channel and edge-MLP shapes the dispatch accepts beyond in = out = 64 and k_in = 6, against the fp64 oracle,
and the fp16 range contract for every 16-bit writer of edge features and kernel matrices.

Every case proves which kernel instantiation ran (torch.profiler kernel names), so that a change of the dispatch cannot
quietly move a case onto a kernel it was not written for.  Errors are max|out - ref| / max|ref|.  pytest -m gpu."""
import ctypes
import re
import time

import pytest
import torch

from oracle import nnconv_oracle as O
from tests.helpers import TOL, DenseNetLike, emulated_nnconv_forward, make_conv, rel_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
STREAM_TOL = 1e-5          # streamed vs cached, same inputs: fp32 scatter order only (tests/test_gpu_stream.py)
# fused persistent kernel vs the per-batch kernels (option no_fuse) on the same cached h: only the order of the fp32
# scatter atomics differs (measured 1.1e-7 .. 2.4e-7 on every f16 / bf16 case below, H100 80GB HBM3, 700 W)
FUSE_TOL = 1e-6
BWD_TC_TOL = {'f16': 3e-3, 'f16x2': 2e-4}    # f16 vs the rounding-consistent forward, f16x2 vs the exact oracle
BWD_FP32_TOL = 2e-4                          # CUDA-core backward vs the exact oracle (DESIGN 5)
FMT = {'f16': 0, 'bf16': 1, 'f16x2': 0}      # template argument FMT of the tensor-core kernels
L1_T = {'f16': '__half', 'bf16': '__nv_bfloat16'}


def _cls():
    from graph_pde_b200.nn_conv import NNConv_old
    return NNConv_old


def _lib_error():
    from graph_pde_b200._lib import NNConvLibraryError
    return NNConvLibraryError


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


@pytest.fixture
def mode(monkeypatch):
    """Set nn_conv._EDGE_KERNELS ('on': formulation B, 'off': formulation C) for one test."""
    from graph_pde_b200 import nn_conv

    def setter(m):
        monkeypatch.setattr(nn_conv, '_EDGE_KERNELS', m)
    setter('off')
    return setter


def _graph(k_in, seed=5, N=300, E=5000):
    """Unsorted sources (the radix-sort plan), a hub with 700 out-edges (several units of one source), ten copies of one
    edge, nodes without in-edges (0..9) and isolated nodes (N-10..N-1)."""
    gen = torch.Generator().manual_seed(seed)
    src = torch.randint(0, N - 20, (E,), generator=gen)
    dst = torch.randint(10, N - 10, (E,), generator=gen)
    src[:700] = 7
    src[1000:1010] = src[1000]
    dst[1000:1010] = dst[1000]
    return torch.stack([src, dst]), torch.randn(E, k_in, generator=gen)


def _params(layers, cin, cout, seed=11):
    torch.manual_seed(seed)
    lin = [m for m in DenseNetLike(layers).layers if isinstance(m, torch.nn.Linear)]
    return ([l.weight.detach().clone() for l in lin], [l.bias.detach().clone() for l in lin],
            torch.randn(cin, cout) * 0.1, torch.randn(cout) * 0.1)


def _oracle(x, ei, ea, ws, bs, root, bias, aggr):
    d = lambda v: None if v is None else v.double()
    return O.nnconv_forward(x.double(), ei, ea.double(), [d(w) for w in ws], [d(b) for b in bs], d(root), d(bias), aggr,
                            x.size(1), ws[-1].size(0) // x.size(1), edge_chunk=1024)


def _launched(fn):
    """fn() under torch.profiler with CUDA activities: its result and the names of the kernels it launched.  Now and
    then a profile comes back without any device record (about one in a few hundred short profiles on an H100); it is
    then taken again: fn is deterministic, and a repeated call launches the kernels of its application again."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    for _ in range(4):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
            time.sleep(0.02)             # let the activity buffers of the kernels just finished reach the profiler
        names = {e.name for e in prof.events() if e.device_type == DeviceType.CUDA}
        if names:
            break
    assert names, 'no device records in four profiles'
    return out, ' | '.join(sorted(names))


def _fused(prec, nc):
    return r'k_apply_tc<%d,\s*64,\s*%d>' % (FMT[prec], nc)


def _conv(prec, nc):
    return r'k_conv_tc<%d,\s*%d>' % (FMT[prec], nc)


def _witness(names, pattern, present=True):
    assert (re.search(pattern, names) is not None) == present, (pattern, names)


# ---- 1. forward, formulation C ----------------------------------------------------------------------------------------
# name: (in, out, edge-MLP widths, what runs at f16 / bf16, what f16x2 does: None = refuses, else what runs)
C_CASES = {
    'nc16': (16, 16, [6, 64, 128, 16 * 16], 'fused', 'fused'),
    'nc48': (48, 48, [6, 64, 128, 48 * 48], 'fused', 'fused'),
    'in1_out64': (1, 64, [6, 64, 128, 64], 'fused', 'fused'),                  # 63 zero-padded Xc columns
    'in128_out32': (128, 32, [6, 64, 128, 128 * 32], 'fused', 'fused'),        # Xc: 2 resident boxes / 6 per stage
    'in256_out16': (256, 16, [6, 64, 128, 256 * 16], 'fused', 'fused'),        # Xc box in every stage
    'out80': (64, 80, [6, 64, 128, 64 * 80], 'conv', None),
    'out96': (32, 96, [6, 64, 128, 32 * 96], 'conv', None),
    'out112': (64, 112, [6, 64, 128, 64 * 112], 'conv', None),
    'out128': (32, 128, [6, 64, 128, 32 * 128], 'conv', None),
    'kp704': (64, 64, [6, 128, 704, 64 * 64], 'fused', None),                  # 11 chunks (33 at f16x2: no schedule)
    'kp1088': (64, 64, [6, 128, 1088, 64 * 64], 'conv', None),                 # 17 chunks: no fused schedule
    'kin24_2layer': (64, 64, [24, 128, 64 * 64], 'fused', None),               # CUDA-core first layer straight into h
    'kin24_3layer': (64, 64, [24, 64, 256, 64 * 64], 'fused', None),           # ... into the ping-pong buffer
    'single_linear': (64, 64, [100, 64 * 64], 'fused', None),                  # identity first layer, Kp = 128
}
_ORACLE_CACHE = {}


def _c_problem(name, aggr):
    cin, cout, layers = C_CASES[name][:3]
    ei, ea = _graph(layers[0])
    ws, bs, root, bias = _params(layers, cin, cout)
    x = torch.randn(300, cin, generator=torch.Generator().manual_seed(2))
    if (name, aggr) not in _ORACLE_CACHE:
        _ORACLE_CACHE[(name, aggr)] = _oracle(x, ei, ea, ws, bs, root, bias, aggr)
    return ei, ea, ws, bs, root, bias, x, _ORACLE_CACHE[(name, aggr)]


@pytest.mark.parametrize('name', list(C_CASES))
@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2'])
def test_formulation_c_shapes(precision, name, mode, monkeypatch, lib_options):
    """Every tensor-core instantiation the dispatch selects for formulation C, both aggregations, against the oracle;
    the fused cases also through the per-batch kernels (no_fuse) and, at NC = 16 / 48, through a Y ring so small that
    about a hundred source batches pass the flag protocol."""
    from graph_pde_b200 import nn_conv
    if name == 'kin24_3layer':
        monkeypatch.setattr(nn_conv, '_EF_WS_BYTES', 1 << 20)        # several chunks of the hidden-layer pass
    cin, cout, layers, path16, path_split = C_CASES[name]
    path = path_split if precision == 'f16x2' else path16
    for aggr in ('mean', 'add'):
        ei, ea, ws, bs, root, bias, x, ref = _c_problem(name, aggr)
        conv = make_conv(_cls(), ws, bs, root, bias, aggr, cin, cout, precision, DEV)
        xd, eid, ead = x.to(DEV), ei.to(DEV), ea.to(DEV)
        if path is None:
            with pytest.raises(_lib_error()):
                with torch.no_grad():
                    conv(xd, eid, ead)
            continue
        prep = conv._get_prepared(precision)
        assert prep.tc
        with torch.no_grad():
            out, names = _launched(lambda: conv(xd, eid, ead))
        assert bool(torch.isfinite(out).all())
        assert rel_err(out, ref) < TOL[precision], (aggr, rel_err(out, ref))
        if aggr != 'mean':
            continue
        _witness(names, _fused(precision, cout) if path == 'fused' else _conv(precision, cout))
        if path == 'conv':
            _witness(names, r'k_apply_tc<', False)
        if layers[0] > 20:
            _witness(names, r'k_edge_layer1<%s>' % L1_T[precision])
        if path == 'fused' and precision != 'f16x2':
            lib_options('no_fuse', 1)
            with torch.no_grad():
                out_nf, names_nf = _launched(lambda: conv(xd, eid, ead))
            lib_options('no_fuse', None)
            _witness(names_nf, _conv(precision, cout))
            print(name, precision, 'fused vs no_fuse', rel_err(out_nf, out))
            assert rel_err(out_nf, out) < FUSE_TOL, rel_err(out_nf, out)
        if cout in (16, 48):
            monkeypatch.setattr(nn_conv, '_Y_BYTES', cout * conv._get_prepared(precision).dims[-2] * 2 * 9)
            with torch.no_grad():
                out_small, names_small = _launched(lambda: conv(xd, eid, ead))
            monkeypatch.setattr(nn_conv, '_Y_BYTES', 0)
            _witness(names_small, _fused(precision, cout))
            assert rel_err(out_small, ref) < TOL[precision]


@pytest.mark.parametrize('precision', ['f16', 'bf16', 'f16x2'])
def test_out_not_a_multiple_of_16_points_at_fp32(precision, mode):
    """out = 40 has no tensor-core schedule: the call raises and names precision fp32, which gets it right."""
    cin, cout, layers = 32, 40, [6, 64, 128, 32 * 40]
    ei, ea = _graph(6)
    ws, bs, root, bias = _params(layers, cin, cout)
    x = torch.randn(300, cin, generator=torch.Generator().manual_seed(2))
    conv = make_conv(_cls(), ws, bs, root, bias, 'mean', cin, cout, precision, DEV)
    with pytest.raises(_lib_error(), match='precision fp32'):
        with torch.no_grad():
            conv(x.to(DEV), ei.to(DEV), ea.to(DEV))
    conv = make_conv(_cls(), ws, bs, root, bias, 'mean', cin, cout, 'fp32', DEV)
    with torch.no_grad():
        out = conv(x.to(DEV), ei.to(DEV), ea.to(DEV))
    assert rel_err(out, _oracle(x, ei, ea, ws, bs, root, bias, 'mean')) < TOL['fp32']


# ---- 2. forward, formulation B (per-edge kernel matrices) ------------------------------------------------------------
def _multipole(s):
    from graph_pde_b200 import graphs
    X, eis, eas = graphs.multi_pole_grid1d(torch.randn(s, generator=torch.Generator().manual_seed(2)), s,
                                           is_periodic=True, levels=2)
    return eis[1], eas[1]


@pytest.mark.parametrize('shape', [(16, 64), (64, 16), (48, 48), (128, 64), (64, 128)])
@pytest.mark.parametrize('precision', ['f16', 'bf16'])
def test_formulation_b_scalar_kernels(precision, shape, mode):
    """The scalar application kernels of formulation B (in/out other than 32x32 and 64x64): warp per source at 4096
    sources with 2-4 out-edges each, warp per edge at 256; plain applications and residual steps."""
    from graph_pde_b200 import nn_conv
    mode('on')
    cin, cout = shape
    for s, kernel in ((4096, r'k_apply_edge_src<'), (256, r'k_apply_edge<')):
        ei, ea = _multipole(s)
        ws, bs, root, bias = _params([4, 64, 64, cin * cout], cin, cout, seed=6)
        x = torch.randn(s, cin, generator=torch.Generator().manual_seed(3))
        conv = make_conv(_cls(), ws, bs, root, bias, 'mean', cin, cout, precision, DEV)
        xd, eid, ead = x.to(DEV), ei.to(DEV), ea.to(DEV)
        n0 = nn_conv.stats.get('edge_kernel_passes', 0)
        with torch.no_grad():
            out, names = _launched(lambda: conv(xd, eid, ead))
        assert nn_conv.stats.get('edge_kernel_passes', 0) == n0 + 1
        _witness(names, kernel)
        _witness(names, r'k_apply_tc<|k_conv_tc<', False)
        assert rel_err(out, _oracle(x, ei, ea, ws, bs, root, bias, 'mean')) < TOL[precision], (s, shape)
        if cin == cout:
            with torch.no_grad():
                z = conv.residual_step(xd, eid, ead, relu_in=True)
            xr = torch.relu(x)
            ref = xr.double() + _oracle(xr, ei, ea, ws, bs, root, bias, 'mean')
            assert rel_err(z, ref) < TOL[precision], (s, shape)


def test_formulation_b_rejected_shape_falls_back_to_c(mode):
    """in * out = 48 is not a multiple of 64: formulation B declines and the fused kernel of formulation C runs."""
    from graph_pde_b200 import nn_conv
    mode('on')
    cin, cout = 3, 16
    ei, ea = _multipole(256)
    ws, bs, root, bias = _params([4, 64, 64, cin * cout], cin, cout, seed=6)
    x = torch.randn(256, cin, generator=torch.Generator().manual_seed(3))
    conv = make_conv(_cls(), ws, bs, root, bias, 'mean', cin, cout, 'f16', DEV)
    n0 = nn_conv.stats.get('edge_kernel_passes', 0)
    with torch.no_grad():
        out, names = _launched(lambda: conv(x.to(DEV), ei.to(DEV), ea.to(DEV)))
    assert nn_conv.stats.get('edge_kernel_passes', 0) == n0
    _witness(names, _fused('f16', 16))
    _witness(names, r'k_apply_edge', False)
    assert rel_err(out, _oracle(x, ei, ea, ws, bs, root, bias, 'mean')) < TOL['f16']


# ---- 3. backward -----------------------------------------------------------------------------------------------------
def _bwd_problem(layers, cin, cout, T=2):
    gen = torch.Generator().manual_seed(17)
    N, E = 150, 2500
    src = torch.randint(0, N - 5, (E,), generator=gen)
    dst = torch.randint(2, N, (E,), generator=gen)
    src[:300] = 3                                    # unsorted sources, a hub with several tiles
    ei = torch.stack([src, dst])
    ea = torch.randn(E, layers[0], generator=gen)
    xs = [torch.randn(N, cin, generator=gen) for _ in range(T)]
    gouts = [torch.randn(N, cout, generator=gen) for _ in range(T)]
    ws, bs, root, bias = _params(layers, cin, cout, seed=3)
    return ei, ea, xs, gouts, ws, bs, root, bias


def _ref_grads(fwd, ea, xs, gouts, ws, bs, root, bias):
    """autograd (fp64, CPU) of sum_t sum(fwd(x_t) * g_t) w.r.t. every x_t, edge_attr and every parameter"""
    lv = {'ea': ea.double(), 'root': root.double(), 'bias': bias.double()}
    for i in range(len(ws)):
        lv['W%d' % i], lv['b%d' % i] = ws[i].double(), bs[i].double()
    lv = {k: v.requires_grad_(True) for k, v in lv.items()}
    xl = [x.double().requires_grad_(True) for x in xs]
    wr = [lv['W%d' % i] for i in range(len(ws))]
    br = [lv['b%d' % i] for i in range(len(ws))]
    sum((fwd(x, lv['ea'], wr, br, lv['root'], lv['bias']) * g.double()).sum() for x, g in zip(xl, gouts)).backward()
    ref = {k: v.grad for k, v in lv.items()}
    ref.update({'x%d' % t: x.grad for t, x in enumerate(xl)})
    return ref


def _run_grads(conv, ei, ea, xs, gouts):
    ead = ea.to(DEV).requires_grad_(True)
    xds = [x.to(DEV).requires_grad_(True) for x in xs]
    eid = ei.to(DEV)
    sum((conv(x, eid, ead) * g.to(DEV)).sum() for x, g in zip(xds, gouts)).backward()
    got = {'x%d' % t: x.grad for t, x in enumerate(xds)}
    for i, l in enumerate([m for m in conv.nn.layers if isinstance(m, torch.nn.Linear)]):
        got['W%d' % i], got['b%d' % i] = l.weight.grad, l.bias.grad
    got['root'], got['bias'], got['ea'] = conv.root.grad, conv.bias.grad, ead.grad
    return got


def _grad_errors(got, ref):
    return {k: rel_err(got[k], ref[k]) for k in ref}


@pytest.mark.parametrize('cin', [1, 16, 48])
@pytest.mark.parametrize('precision', ['f16', 'f16x2'])
def test_tc_backward_narrow_inputs(precision, cin, mode):
    """Tensor-core backward with in < 64, T = 2 applications sharing the conv: x, every parameter and edge_attr."""
    cout, layers = 64, [6, 64, 128, cin * 64]
    ei, ea, xs, gouts, ws, bs, root, bias = _bwd_problem(layers, cin, cout)
    if precision == 'f16':
        fwd = lambda x, e, w, b, r, bb: emulated_nnconv_forward(x, ei, e, w, b, r, bb, 'mean', 'f16', edge_chunk=500)
    else:
        fwd = lambda x, e, w, b, r, bb: O.nnconv_forward(x, ei, e, w, b, r, bb, 'mean', cin, cout, edge_chunk=500)
    ref = _ref_grads(fwd, ea, xs, gouts, ws, bs, root, bias)
    conv = make_conv(_cls(), ws, bs, root, bias, 'mean', cin, cout, precision, DEV)
    assert conv._get_prepared(precision).bwd_tc
    errs = _grad_errors(_run_grads(conv, ei, ea, xs, gouts), ref)
    assert max(errs.values()) < BWD_TC_TOL[precision], errs


@pytest.mark.parametrize('layers,cin,cout', [
    ([6, 64, 128, 128 * 64], 128, 64),
    ([6, 64, 128, 64 * 128], 64, 128),
    ([6, 64, 128, 48 * 48], 48, 48),
    ([24, 128, 64 * 64], 64, 64),
])
def test_cuda_core_backward_after_16_bit_forward(layers, cin, cout, mode):
    """Shapes the tensor-core backward does not cover train through the fp32 CUDA-core backward after a 16-bit forward."""
    ei, ea, xs, gouts, ws, bs, root, bias = _bwd_problem(layers, cin, cout)
    fwd = lambda x, e, w, b, r, bb: O.nnconv_forward(x, ei, e, w, b, r, bb, 'mean', cin, cout, edge_chunk=500)
    ref = _ref_grads(fwd, ea, xs, gouts, ws, bs, root, bias)
    conv = make_conv(_cls(), ws, bs, root, bias, 'mean', cin, cout, 'f16', DEV)
    assert not conv._get_prepared('f16').bwd_tc
    errs = _grad_errors(_run_grads(conv, ei, ea, xs, gouts), ref)
    assert max(errs.values()) < BWD_FP32_TOL, errs


# ---- 4. streamed edge features -----------------------------------------------------------------------------------------
def _h_bytes(conv, ei, n, precision):
    from graph_pde_b200 import _lib, nn_conv
    plan = nn_conv.get_plan(ei, n, conv.flow)
    prep = conv._get_prepared(precision)
    h_b, ws_b = ctypes.c_size_t(), ctypes.c_size_t()
    _lib.check(_lib.lib().nnconv_edge_features_sizes(plan.handle, prep.handle, 1 << 20, ctypes.byref(h_b),
                                                     ctypes.byref(ws_b)))
    return h_b.value


def _apply_t(conv, xs, ei, ea, budget):
    from graph_pde_b200 import nn_conv
    conv.edge_feature_bytes = budget
    conv.invalidate()
    c0 = nn_conv.stats['streamed_chunk_passes']
    with torch.no_grad():
        outs = [conv(x, ei, ea) for x in xs]
    return outs, nn_conv.stats['streamed_chunk_passes'] - c0


@pytest.mark.parametrize('precision,cin,cout,layers,kernel', [
    ('f16', 48, 48, [6, 128, 128, 48 * 48], _fused('f16', 48)),          # fused kernel over unit ranges
    ('f16', 32, 128, [6, 128, 128, 32 * 128], _conv('f16', 128)),        # per-batch kernels over unit ranges
    ('f16x2', 128, 32, [6, 128, 128, 128 * 32], _fused('f16x2', 32)),    # Xc box per stage over unit ranges
    ('f16', 64, 64, [24, 128, 64 * 64], r'k_edge_layer1<__half>'),      # first layer straight into each chunk's h
])
def test_streamed_shapes(precision, cin, cout, layers, kernel, monkeypatch, mode):
    """Budget 0 and half of h resident against the cached run on the same inputs (T = 2), and against the oracle."""
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_EF_WS_BYTES', 3 << 20)
    ei, ea = _graph(layers[0])
    ws, bs, root, bias = _params(layers, cin, cout)
    gen = torch.Generator().manual_seed(2)
    xs = [torch.randn(300, cin, generator=gen) for _ in range(2)]
    conv = make_conv(_cls(), ws, bs, root, bias, 'mean', cin, cout, precision, DEV)
    eid, ead, xds = ei.to(DEV), ea.to(DEV), [x.to(DEV) for x in xs]
    cached, n = _apply_t(conv, xds, eid, ead, None)
    assert n == 0
    for k, x in enumerate(xs):
        assert rel_err(cached[k], _oracle(x, ei, ea, ws, bs, root, bias, 'mean')) < TOL[precision]
    hb = _h_bytes(conv, eid, 300, precision)
    for budget in (0, hb // 2):
        (got, n), names = _launched(lambda: _apply_t(conv, xds, eid, ead, budget))
        assert n >= 2, (budget, n)
        _witness(names, kernel)
        for k in range(2):
            assert rel_err(got[k], cached[k]) < STREAM_TOL, (budget, k, rel_err(got[k], cached[k]))


# ---- 5. the fp16 range contract ----------------------------------------------------------------------------------------
def _overflow_problem(layers, scale_w1=1.0, ea_scale=1.0, cin=64, cout=64):
    ei, ea = _graph(layers[0])
    ws, bs, root, bias = _params(layers, cin, cout)
    ws[0], bs[0] = ws[0] * scale_w1, bs[0] * scale_w1
    x = torch.randn(300, cin, generator=torch.Generator().manual_seed(2))
    return ei, ea * ea_scale, ws, bs, root, bias, x


@pytest.mark.parametrize('case', ['kin24_2layer', 'kin24_3layer', 'kin24_3layer_nan', 'single_linear',
                                  'kin24_2layer_streamed'])
def test_fp16_range_of_every_first_layer_writer(case, mode):
    """A first layer whose 16-bit output leaves the fp16 range raises FloatingPointError at f16, while bf16 stays finite
    and within its tolerance of the oracle.  kin24_3layer_nan: hidden units 0 and 1 are one unit written twice, scaled
    past the range, with opposite weights in the next layer -- that layer's GEMM sees inf - inf = NaN in every output
    and its ReLU turns the NaN into 0 before its own range check, so only the writer of the first layer can tell."""
    if case.startswith('kin24_2layer'):
        problem = _overflow_problem([24, 128, 64 * 64], scale_w1=3e5)
    elif case == 'kin24_3layer':
        problem = _overflow_problem([24, 64, 256, 64 * 64], scale_w1=3e5)
    elif case == 'kin24_3layer_nan':
        problem = _overflow_problem([24, 64, 256, 64 * 64])
        ws, bs = problem[2], problem[3]
        ws[0][:2], bs[0][:2] = ws[0][0] * 1e5, bs[0][0] * 1e5
        ws[1][:, 1] = -ws[1][:, 0]
    else:
        problem = _overflow_problem([16, 64 * 64], ea_scale=3e5)
    ei, ea, ws, bs, root, bias, x = problem
    budget = 0 if case.endswith('streamed') else None
    ref = _oracle(x, ei, ea, ws, bs, root, bias, 'mean')
    for precision in ('f16', 'bf16'):
        conv = make_conv(_cls(), ws, bs, root, bias, 'mean', 64, 64, precision, DEV)
        conv.edge_feature_bytes = budget
        if precision == 'f16':
            with pytest.raises(FloatingPointError):
                with torch.no_grad():
                    conv(x.to(DEV), ei.to(DEV), ea.to(DEV))
                    torch.cuda.synchronize()
        else:
            with torch.no_grad():
                out = conv(x.to(DEV), ei.to(DEV), ea.to(DEV))
            assert bool(torch.isfinite(out).all())
            assert rel_err(out, ref) < TOL['bf16'], rel_err(out, ref)


@pytest.mark.parametrize('precision', ['f16', 'bf16'])
def test_large_last_layer_bias_in_both_formulations(precision, mode):
    """b_L ~ 1e5 with every |h| and |Y| inside the fp16 range: formulation C carries b_L in fp32 (x . B3); formulation B
    rounds K_e = W_L h_e + b_L to 16 bits, and at f16 it must not hand back inf: the build of K_e counts values beyond
    the fp16 range and the application falls back to formulation C."""
    from graph_pde_b200 import nn_conv
    cin = cout = 64
    ei, ea = _multipole(256)
    ws, bs, root, bias = _params([4, 64, 64, cin * cout], cin, cout, seed=6)
    bs[-1] = bs[-1] + 1e5
    x = torch.randn(256, cin, generator=torch.Generator().manual_seed(3))
    ref = _oracle(x, ei, ea, ws, bs, root, bias, 'mean')
    xd, eid, ead = x.to(DEV), ei.to(DEV), ea.to(DEV)
    outs = {}
    for m in ('off', 'on', 'auto'):
        mode(m)
        conv = make_conv(_cls(), ws, bs, root, bias, 'mean', cin, cout, precision, DEV)
        n0 = nn_conv.stats.get('edge_kernel_passes', 0)
        with torch.no_grad():
            outs[m], names = _launched(lambda: conv(xd, eid, ead))
            again = conv(xd, eid, ead)                                # the cached decision
        assert bool(torch.isfinite(outs[m]).all()), m
        assert torch.equal(again, outs[m]) or rel_err(again, outs[m]) < 1e-6, m
        assert nn_conv.stats.get('edge_kernel_passes', 0) == n0 + (m != 'off'), m
        b_ran = m != 'off' and precision == 'bf16'
        _witness(names, r'k_apply_edge', b_ran)
        _witness(names, _fused(precision, cout), not b_ran)
    assert rel_err(outs['off'], ref) < TOL[precision]
    for m in ('on', 'auto'):
        assert rel_err(outs[m], outs['off']) < 2 * TOL[precision], m
