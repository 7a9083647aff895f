"""Every application schedule of the library, bit for bit, on the exact probes (tests/probes.py).

The knobs of csrc/options.h choose which code computes an application: the fused persistent kernel or the per-batch
Y-GEMM and contraction kernels, how they are launched, the scatter epilogue, the GEMM store path, the passes over the
B-slot ring, the Y ring's depth and batch shape, and the pipeline depths.  Each knob is classified once below:
``SCHEDULES`` changes which code runs, ``RESULT_NEUTRAL`` changes only cache hints or bookkeeping, ``EXCLUDED`` is
wrong by design, instrumentation, or changes device-wide state.  ``test_every_knob_is_classified_once`` reads the
option table of csrc/options.cu, so a knob added later cannot skip this matrix.

On an add-exact probe every schedule must equal fp64 bit for bit, so a schedule that loses, doubles or misroutes one
edge fails at the node it touches.  The forward matrix is an explicit pairwise cover (``COVER``, written out as a
table below): every schedule meets every feature once, at a precision that rotates through the precisions the
schedule exists at.  ``BACKWARD_COVER`` runs a training step after the forward under each schedule.

A knob that a precision does not have (the per-batch kernels at f16x2) is ignored there: the answer and the launch
count equal the default schedule's (``test_per_batch_knobs_are_ignored_at_f16x2``).

GPU tests: pytest -m gpu.  The classification and the cover are checked without a GPU."""
import os
import re

import pytest
import torch

from tests import act_oracle as A
from tests import act_probe as AP
from tests import bipartite_oracle as BO
from tests import probes as P
from tests import test_gpu_aggr_max as AM
from tests import test_gpu_bipartite as BP
from tests import test_gpu_edge_activation as EA
from tests import test_gpu_edge_activation_more as EAM
from tests import test_gpu_exact_backward as EB
from tests import test_gpu_exact_forward as EF

DEV = 'cuda:0'
ALL = ('f16', 'bf16', 'f16x2')
CHAIN = ('f16', 'bf16')             # the per-batch kernels: f16x2 runs in the fused kernel only

# Y bytes of one source of the mixed probe (out 64 x Kp 128 x 2 bytes; twice that at f16x2)
_Y_SRC = 64 * 128 * 2

# ---- 1. the knobs --------------------------------------------------------------------------------------------------
# name: (library options, nn_conv module settings, precisions the schedule exists at).  A module setting `_Y_BYTES` is
# doubled at f16x2, whose Y rows are (hi, lo) pairs.
SCHEDULES = {
    'fused_coop': ({}, {}, ALL),
    'fused_no_coop': ({'no_coop': 1}, {}, ALL),
    'per_batch_pdl': ({'no_fuse': 1}, {}, CHAIN),
    'per_batch_stream_order': ({'no_fuse': 1, 'no_pipe': 1}, {}, CHAIN),
    'per_batch_many_batches': ({'no_fuse': 1}, {'_Y_BYTES': 3 * 4 * _Y_SRC}, CHAIN),
    # one Y buffer for every batch: each batch's Y GEMM must wait for the previous batch's contraction
    'per_batch_stream_order_many_batches': ({'no_fuse': 1, 'no_pipe': 1}, {'_Y_BYTES': 3 * 4 * _Y_SRC}, CHAIN),
    'scatter_mode0': ({'scatter_mode': 0}, {}, ALL),
    'gemm_direct_store': ({'gemm_direct_store': 1}, {}, ALL),
    # forced pass counts: 2 and 3 passes where Kp / 64 has them with >= 4 B slots per pass (hub_batches at f16x2),
    # ignored elsewhere
    'apply_passes2': ({'apply_passes': 2}, {}, ALL),
    'apply_passes3': ({'apply_passes': 3}, {}, ALL),
    'many_flag_batches': ({}, {'_Y_BYTES': 3 * 4 * _Y_SRC}, ALL),
    'ring2': ({'ring': 2}, {'_Y_BYTES': 2 * 8 * _Y_SRC}, ALL),
    'ring8': ({'ring': 8}, {'_Y_BYTES': 8 * 4 * _Y_SRC}, ALL),
    # batches of 128 sources in a deeper ring once the Y budget holds more than 3 x 128 sources: the bipartite probe's
    # 697 sources (5 slots); the smaller probes keep the default geometry
    'ring_deep': ({'ring_deep': 1}, {}, ALL),
    # the A-stage caps take effect from 2 (0 and 1 leave the automatic depth)
    'apply_stages2': ({'apply_stages': 2}, {}, ALL),
    'conv_stages2': ({'no_fuse': 1, 'conv_stages': 2}, {}, CHAIN),
    'conv_one_per_sm': ({'no_fuse': 1, 'conv_one_per_sm': 1}, {}, CHAIN),
    # two layers at once.  scatter_mode switches the fused kernel's epilogue only, so it is paired with a fused knob.
    'no_fuse+gemm_direct_store': ({'no_fuse': 1, 'gemm_direct_store': 1}, {}, CHAIN),
    'no_coop+gemm_direct_store': ({'no_coop': 1, 'gemm_direct_store': 1}, {}, ALL),
    'scatter_mode0+ring2': ({'scatter_mode': 0, 'ring': 2}, {'_Y_BYTES': 2 * 8 * _Y_SRC}, ALL),
}

# name: (the values other than the default, why the result cannot depend on it)
RESULT_NEUTRAL = {
    'tmap_promo': ((0, 1), 'L2 promotion of the operand tensor maps: a cache hint of the TMA loads'),
    'y_store_policy': ((1, 2), 'L2 eviction hint of the fused kernel\'s Y stores'),
    'apply_a_policy': ((1,), 'L2 eviction hint of the fused kernel\'s h stream'),
    'gemm_b_policy': ((0,), 'L2 eviction hint of the GEMM\'s weight tiles'),
    'overflow_check': ((0,), 'only whether the 16-bit writers count fp16 overflows; the values they store are the same'),
}

EXCLUDED = {
    'debug_scatter': 'timing experiment of the fused kernel\'s scatter: wrong results by design',
    'trace': 'instrumentation: CTA timeline records',
    'conv_debug': 'instrumentation of the per-batch conv kernel',
    'l2_persist': 'sets the context\'s persisting-L2 carve-out, device state shared with every other process',
    'l2_reset': 'resets the context\'s persisting-L2 lines, device state shared with every other process',
}

_OPTIONS_CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'graph_pde_b200', 'csrc',
                           'options.cu')


def knob_names(options_cu_text):
    """The option names of the kEntries table of csrc/options.cu."""
    table = options_cu_text.split('kEntries[]', 1)[1].split('};', 1)[0]
    return re.findall(r'\{\s*"([a-z0-9_]+)"\s*,\s*"NNCONV_', table)


def misclassified(options_cu_text):
    """{knob: number of classes it is in} for every knob not in exactly one class, and every classified name that is
    not a knob (count -1)."""
    in_schedules = {k for opts, _, _ in SCHEDULES.values() for k in opts}
    names = knob_names(options_cu_text)
    bad = {}
    for n in names:
        c = (n in in_schedules) + (n in RESULT_NEUTRAL) + (n in EXCLUDED)
        if c != 1:
            bad[n] = c
    for n in in_schedules | set(RESULT_NEUTRAL) | set(EXCLUDED):
        if n not in names:
            bad[n] = -1
    return bad


def test_every_knob_is_classified_once():
    with open(_OPTIONS_CU) as f:
        text = f.read()
    assert len(knob_names(text)) >= 21
    assert misclassified(text) == {}


def test_the_guard_reports_an_unclassified_knob():
    with open(_OPTIONS_CU) as f:
        text = f.read()
    dummy = text.replace('    {"no_fuse",', '    {"dummy_knob", "NNCONV_DUMMY_KNOB", &Options::no_fuse, 0},\n    {"no_fuse",', 1)
    assert dummy != text
    assert misclassified(dummy) == {'dummy_knob': 0}


# ---- 2. the cover ----------------------------------------------------------------------------------------------------
# feature: (aggregations, graph kind, edge-network activation, edge-feature residency)
FEATURES = {
    'add': (('add',), 'square', 'relu', 'cached'),
    'mean': (('mean',), 'square', 'relu', 'cached'),
    'max': (('max',), 'square', 'relu', 'cached'),
    'hub_batches': (('add', 'mean'), 'square', 'relu', 'cached'),
    'partial_tiles': (('add', 'mean'), 'square', 'relu', 'cached'),
    'bipartite': (('add', 'max'), 'bipartite', 'relu', 'cached'),
    'bipartite_size': (('mean',), 'bipartite', 'relu', 'cached'),
    'leaky_relu': (('add',), 'square', 'leaky_relu', 'cached'),
    'relu6_bound': (('max',), 'square', 'relu6', 'cached'),
    'hardtanh_bound': (('max',), 'square', 'hardtanh', 'cached'),
    'streamed_0': (('add',), 'square', 'relu', 'streamed'),
    'streamed_straddle': (('add',), 'square', 'relu', 'streamed'),
    'residual': (('add',), 'square', 'relu', 'cached'),
}


def _cover():
    """Schedule i meets feature j at precision precs_i[(i + j) mod len(precs_i)]: every schedule meets every feature,
    and, since there are more features than precisions, every precision it exists at."""
    cases = []
    for i, (s, (_, _, precs)) in enumerate(SCHEDULES.items()):
        for j, f in enumerate(FEATURES):
            cases.append((s, f, precs[(i + j) % len(precs)]))
    return cases


COVER = _cover()


def _backward_cover():
    """Per schedule: add with kept activations, max with recomputed ones (the tensor-core backward, at precisions
    rotating through the schedule's), and the CUDA-core backward after an f16 forward, add and max alternating."""
    cases = []
    for i, (s, (_, _, precs)) in enumerate(SCHEDULES.items()):
        cases.append((s, 'add', 'kept', 'tc', precs[i % len(precs)]))
        cases.append((s, 'max', 'recomputed', 'tc', precs[(i + 1) % len(precs)]))
        cases.append((s, ('add', 'max')[i % 2], 'kept', 'fp32', 'f16'))
    return cases


BACKWARD_COVER = _backward_cover()

_ABBR = {'f16': 'h', 'bf16': 'b', 'f16x2': 'x'}


def cover_table():
    """The forward cover as text: one row per schedule, one column per feature (h = f16, b = bf16, x = f16x2)."""
    feats = list(FEATURES)
    at = {(s, f): pr for s, f, pr in COVER}
    w = max(len(s) for s in SCHEDULES)
    lines = ['%-*s  %s' % (w, '', ' '.join('%d' % (j % 10) for j in range(len(feats))))]
    for s in SCHEDULES:
        lines.append('%-*s  %s' % (w, s, ' '.join(_ABBR[at[s, f]] for f in feats)))
    lines.append('columns: ' + ', '.join('%d %s' % (j, f) for j, f in enumerate(feats)))
    return lines


# The forward cover, as cover_table() renders it (test_cover_table_is_written_out keeps it current):
#                                      0 1 2 3 4 5 6 7 8 9 0 1 2
# fused_coop                           h b x h b x h b x h b x h
# fused_no_coop                        b x h b x h b x h b x h b
# per_batch_pdl                        h b h b h b h b h b h b h
# per_batch_stream_order               b h b h b h b h b h b h b
# per_batch_many_batches               h b h b h b h b h b h b h
# per_batch_stream_order_many_batches  b h b h b h b h b h b h b
# scatter_mode0                        h b x h b x h b x h b x h
# gemm_direct_store                    b x h b x h b x h b x h b
# apply_passes2                        x h b x h b x h b x h b x
# apply_passes3                        h b x h b x h b x h b x h
# many_flag_batches                    b x h b x h b x h b x h b
# ring2                                x h b x h b x h b x h b x
# ring8                                h b x h b x h b x h b x h
# ring_deep                            b x h b x h b x h b x h b
# apply_stages2                        x h b x h b x h b x h b x
# conv_stages2                         b h b h b h b h b h b h b
# conv_one_per_sm                      h b h b h b h b h b h b h
# no_fuse+gemm_direct_store            b h b h b h b h b h b h b
# no_coop+gemm_direct_store            h b x h b x h b x h b x h
# scatter_mode0+ring2                  b x h b x h b x h b x h b
# columns: 0 add, 1 mean, 2 max, 3 hub_batches, 4 partial_tiles, 5 bipartite, 6 bipartite_size, 7 leaky_relu, 8 relu6_bound, 9 hardtanh_bound, 10 streamed_0, 11 streamed_straddle, 12 residual


def test_cover_table_is_written_out():
    with open(os.path.abspath(__file__).replace('.pyc', '.py')) as f:
        text = f.read()
    block = text.split('# The forward cover, as cover_table() renders it', 1)[1].split('\n\n', 1)[0]
    written = [l[2:] for l in block.split('\n')[1:]]
    assert written == cover_table()


def test_cover_pairs_every_schedule_with_every_axis():
    """Each schedule meets add, mean and max; square and bipartite graphs; every probe activation; cached and streamed
    edge features; forward and backward; and every precision it exists at."""
    axes = {'aggr': {'add', 'mean', 'max'}, 'graph': {'square', 'bipartite'},
            'act': {'relu', 'leaky_relu', 'relu6', 'hardtanh'}, 'residency': {'cached', 'streamed'}}
    for s, (_, _, precs) in SCHEDULES.items():
        seen = {k: set() for k in axes}
        seen['precision'] = set()
        for s2, f, pr in COVER:
            if s2 != s:
                continue
            aggrs, graph, act, res = FEATURES[f]
            seen['aggr'] |= set(aggrs)
            seen['graph'].add(graph)
            seen['act'].add(act)
            seen['residency'].add(res)
            seen['precision'].add(pr)
        for k, want in axes.items():
            assert seen[k] == want, (s, k, seen[k])
        assert seen['precision'] == set(precs), s
        bwd = [c for c in BACKWARD_COVER if c[0] == s]
        assert {c[1] for c in bwd} == {'add', 'max'} and {c[2] for c in bwd} == {'kept', 'recomputed'}
        assert {c[3] for c in bwd} == {'tc', 'fp32'}, s
    for f in FEATURES:             # and every feature meets every precision
        assert {pr for _, f2, pr in COVER if f2 == f} == set(ALL), f


# ---- fixtures ----------------------------------------------------------------------------------------------------------
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
def formulation_c(monkeypatch):
    from graph_pde_b200 import nn_conv
    monkeypatch.setattr(nn_conv, '_EDGE_KERNELS', 'off')


def _apply(schedule, precision, lib_options, monkeypatch):
    from graph_pde_b200 import nn_conv
    opts, mods, _ = SCHEDULES[schedule]
    for k, v in opts.items():
        lib_options(k, v)
    for k, v in mods.items():
        monkeypatch.setattr(nn_conv, k, v * (2 if k == '_Y_BYTES' and precision == 'f16x2' else 1))


# ---- 3. the forward features ---------------------------------------------------------------------------------------
def _mixed(precision):
    p = P.probe(P.FORWARD, 'mixed', precision=precision)
    return p, bool(P.wide_options(P.FORWARD, 'mixed', precision))


def _f_add_mean(aggr):
    def run(precision, mods, monkeypatch):
        p, wide = _mixed(precision)
        ref, msg = EF._reference(p, aggr, key=('mixed', aggr, wide))
        out, _ = EF._run(p, precision, aggr)
        EF.assert_matches(out, p, aggr, ref, msg)
    return run


_MAX_REF = {}


def _f_max(precision, mods, monkeypatch):
    p, wide = _mixed(precision)
    if wide not in _MAX_REF:
        _MAX_REF[wide] = AM._reference(p)
    out, am, _ = AM._run(p, precision)
    AM._assert_exact(out, am, *_MAX_REF[wide])


def _f_graph(name):
    def run(precision, mods, monkeypatch):
        from graph_pde_b200 import nn_conv
        if name == 'hub_batches' and '_Y_BYTES' not in mods:       # ~100 flag batches, as in test_graphs
            monkeypatch.setattr(nn_conv, '_Y_BYTES', 3 * 4 * 64 * 256 * 2 * (2 if precision == 'f16x2' else 1))
        p = P.probe(P.FORWARD, name, precision=precision)
        wide = bool(P.wide_options(P.FORWARD, name, precision))
        for aggr in ('add', 'mean'):
            ref, msg = EF._reference(p, aggr, key=(name, aggr, wide))
            out, _ = EF._run(p, precision, aggr)
            EF.assert_matches(out, p, aggr, ref, msg)
    return run


_BIP = {}
_N_SRC, _N_DST = 700, 260


def _bipartite_probe(precision):
    """The union probe of test_gpu_bipartite (in-degrees 0 or powers of two up to 16: mean is exact too), proved at
    ``precision``."""
    if precision not in _BIP:
        ei = BP.pow2_bip_graph(_N_SRC, _N_DST, 11)
        union = torch.stack([ei[0], ei[1] + _N_SRC])
        p = P.make_probe(union, _N_SRC + _N_DST, [6, 64, 128, 64 * 64], 64, 64, seed=11)
        P.assert_exact(p, precision, aggr='mean')
        _BIP[precision] = (ei, p, {})
    return _BIP[precision]


def _f_bipartite(with_x_dst):
    def run(precision, mods, monkeypatch):
        from graph_pde_b200.nn_conv import NNConv_old
        ei, p, refs = _bipartite_probe(precision)
        xs, xd = p.x[0][:_N_SRC], p.x[0][_N_SRC:]
        for aggr in (('add', 'max') if with_x_dst else ('mean',)):
            key = (aggr, with_x_dst)
            if key not in refs:
                refs[key] = BO.bipartite_forward(xs, xd if with_x_dst else None, ei, p.ea.double(), p.ws, p.bs, p.root,
                                                 p.bias, aggr, _N_DST)
            conv = p.conv(NNConv_old, precision, aggr, DEV)
            with torch.no_grad():
                if with_x_dst:
                    out = conv((xs.float().to(DEV), xd.float().to(DEV)), ei.to(DEV), p.ea.to(DEV))
                else:
                    out = conv((xs.float().to(DEV), None), ei.to(DEV), p.ea.to(DEV), size=(_N_SRC, _N_DST))
            bad = (out.double().cpu() != refs[key]).any(1)
            assert not bool(bad.any()), (aggr, 'targets differ', torch.nonzero(bad).flatten()[:20].tolist())
    return run


_LEAKY = {}


def _f_leaky_relu(precision, mods, monkeypatch):
    """The exact LeakyReLU(0.25) probe: both applications equal fp64 bit for bit."""
    if precision not in _LEAKY:
        ei, n = AP.graph()
        pr = AP.make(ei, n, precision=precision)
        refs = [A.nnconv_forward(x, ei, pr.ea.double(), pr.ws, pr.bs, pr.root, pr.bias, 'add', 'leaky_relu',
                                 AP.SLOPE)[0] for x in pr.x]
        _LEAKY[precision] = (ei, pr, refs)
    ei, pr, refs = _LEAKY[precision]
    conv = EA._probe_conv(pr, precision)
    with torch.no_grad():
        for t, (x, ref) in enumerate(zip(pr.x, refs)):
            out = conv(x.float().to(DEV), ei.to(DEV), pr.ea.float().to(DEV))
            bad = (out.double().cpu() != ref).any(1)
            assert not bool(bad.any()), (t, 'nodes differ', torch.nonzero(bad).flatten()[:20].tolist())


_BOUND = {}


def _bound_run(kind, p, precision):
    """The clamps' bound probe of test_gpu_edge_activation_more (hidden units whose pre-activation is exactly at, one
    ulp inside and beyond each bound) under aggr='max': (h, out, argmax).  max picks one message per (node, channel),
    so unlike add on these random values it does not depend on the order in which edges reach a node."""
    ei, n = EA._hub_graph(e=6000, hub=2000)
    ea, xs, _ = EA._inputs(ei, n, T=1)
    conv = EAM._bound_probe_conv(kind, p, precision)
    conv.aggr = 'max'
    with torch.no_grad():
        out, am = conv._forward_impl(xs[0].to(DEV), ei.to(DEV), ea.to(DEV), with_argmax=True)
    h = next(iter(conv._h_cache.values())).h
    # the valid rows of the chunk-major h, [64-column panels][E rounded up to 128 rows][64]: what the padding rows hold
    # depends on the store path (the TMA store fills them, st.global leaves them), and no kernel reads them
    e = ei.size(1)
    e_pad = (e + 127) // 128 * 128
    panels = h.numel() // (e_pad * 128)
    h = h[:panels * e_pad * 128].view(torch.int16).view(panels, e_pad, 64)[:, :e]
    return h.cpu(), out.cpu(), am.cpu()


def _bound_baseline(kind, p, precision):
    """The default schedule's (h, out, argmax); computed before the schedule's options are set."""
    if (kind, precision) not in _BOUND:
        _BOUND[kind, precision] = _bound_run(kind, p, precision)
    return _BOUND[kind, precision]


def _f_bound(kind, p):
    def run(precision, mods, monkeypatch):
        h0, out0, am0 = _BOUND[kind, precision]
        h, out, am = _bound_run(kind, p, precision)
        assert torch.equal(h, h0), 'edge features differ from the default schedule\'s'
        bad = (out != out0).any(1) | (am != am0).any(1)
        assert not bool(bad.any()), ('nodes differ from the default schedule', torch.nonzero(bad).flatten()[:20].tolist())
    return run


def _f_streamed(which):
    def run(precision, mods, monkeypatch):
        """test_streamed_edge_features: budget 0, or a resident prefix that ends inside the hub source's units, with
        chunks that end inside the hub; bitwise equal to fp64 and to the cached run of the same schedule."""
        from graph_pde_b200 import nn_conv
        monkeypatch.setattr(nn_conv, '_EF_WS_BYTES', 300007)
        p, wide = _mixed(precision)
        ref, msg = EF._reference(p, 'add', key=('mixed', 'add', wide))
        cached, conv = EF._run(p, precision, 'add')
        EF.assert_matches(cached, p, 'add', ref, msg)
        budget = 0
        if which == 'straddle':
            hb = EF._h_bytes(conv, p)
            counts = torch.bincount(p.src_dst()[0].cpu(), minlength=p.n_nodes)
            hub = int(counts.argmax())
            g_hub, deg_hub = int(counts[:hub].sum()), int(counts[hub])
            budget = (g_hub + deg_hub - 1) * (hb // ((p.ei.size(1) + 127) // 128 * 128))
        c0 = nn_conv.stats['streamed_chunk_passes']
        out, conv = EF._run(p, precision, 'add', edge_feature_bytes=budget)
        assert nn_conv.stats['streamed_chunk_passes'] > c0
        if which == 'straddle':
            e_res = next(iter(conv._h_cache.values())).E_res
            assert g_hub < e_res < g_hub + deg_hub, (g_hub, deg_hub, e_res)
        assert torch.equal(out, cached)
        EF.assert_matches(out, p, 'add', ref, msg)
    return run


def _f_residual(precision, mods, monkeypatch):
    EF._residual(P.probe(P.FORWARD, 'mixed'), precision)


RUNNERS = {
    'add': _f_add_mean('add'),
    'mean': _f_add_mean('mean'),
    'max': _f_max,
    'hub_batches': _f_graph('hub_batches'),
    'partial_tiles': _f_graph('partial_tiles'),
    'bipartite': _f_bipartite(True),
    'bipartite_size': _f_bipartite(False),
    'leaky_relu': _f_leaky_relu,
    'relu6_bound': _f_bound('relu6', None),
    'hardtanh_bound': _f_bound('hardtanh', (-0.3, 0.7)),
    'streamed_0': _f_streamed('0'),
    'streamed_straddle': _f_streamed('straddle'),
    'residual': _f_residual,
}
_BOUND_KIND = {'relu6_bound': ('relu6', None), 'hardtanh_bound': ('hardtanh', (-0.3, 0.7))}


@pytest.mark.gpu
@pytest.mark.parametrize('schedule,feature,precision', COVER, ids=['-'.join(c) for c in COVER])
def test_forward_matrix(schedule, feature, precision, lib_options, monkeypatch, formulation_c):
    if feature in _BOUND_KIND:
        _bound_baseline(*_BOUND_KIND[feature], precision)
    _apply(schedule, precision, lib_options, monkeypatch)
    RUNNERS[feature](precision, SCHEDULES[schedule][1], monkeypatch)


# ---- 4. the backward after each forward schedule ----------------------------------------------------------------------
_MAX_GRAD_REF = {}


@pytest.mark.gpu
@pytest.mark.parametrize('schedule,aggr,acts,mode,precision', BACKWARD_COVER,
                         ids=['-'.join(c) for c in BACKWARD_COVER])
def test_backward_matrix(schedule, aggr, acts, mode, precision, lib_options, monkeypatch, formulation_c):
    """A training step (T = 2 applications of one conv) on the exact backward probe, forward and backward under the
    schedule: x, edge_attr, every Linear, root and bias equal fp64 autograd bit for bit.  Under max the backward routes
    by the argmax its forward produced, so a schedule that picks another winner fails in the gradients."""
    from graph_pde_b200 import nn_conv
    _apply(schedule, precision, lib_options, monkeypatch)
    monkeypatch.setattr(nn_conv, '_BWD_MODE', mode)
    if acts == 'recomputed':
        monkeypatch.setattr(nn_conv, '_KEEP_ACTS_MAX_BYTES', 0)
    p = P.probe(P.BACKWARD, 'mixed', precision=precision)
    b0 = nn_conv.stats['mlp_backwards']
    if aggr == 'add':
        EB.assert_grads_equal(EB._library(p, precision), EB._reference(p, ('mixed', precision, 'x')))
    else:
        if precision not in _MAX_GRAD_REF:
            _MAX_GRAD_REF[precision] = AM._flat(AM._grad_reference(p))
        got = AM._flat(AM._grad_library(p, precision))
        for (k, a), (_, b) in zip(got, _MAX_GRAD_REF[precision]):
            assert torch.equal(a, b), (k, float((a - b).abs().max()))
    assert (nn_conv.stats['mlp_backwards'] > b0) == (mode == 'tc')


# ---- 5. the result-neutral knobs --------------------------------------------------------------------------------------
NEUTRAL_CASES = [(k, v) for k, (vals, _) in RESULT_NEUTRAL.items() for v in vals]
_DEFAULT = {}


def _neutral_run(precision):
    """(add output, max output and argmax, add gradients) of the mixed probes."""
    p, _ = _mixed(precision)
    add, _ = EF._run(p, precision, 'add')
    mx, am, _ = AM._run(p, precision)
    pb = P.probe(P.BACKWARD, 'mixed', precision=precision)
    g = EB._library(pb, precision)
    return p, pb, add.cpu(), mx.cpu(), am.cpu(), {k: v.detach().cpu() for k, v in g.items()}


@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['f16', 'f16x2'])
@pytest.mark.parametrize('knob,value', NEUTRAL_CASES, ids=['%s=%d' % c for c in NEUTRAL_CASES])
def test_result_neutral_knobs(knob, value, precision, lib_options, formulation_c):
    if precision not in _DEFAULT:
        _DEFAULT[precision] = _neutral_run(precision)
    p, pb, add0, mx0, am0, g0 = _DEFAULT[precision]
    wide = bool(P.wide_options(P.FORWARD, 'mixed', precision))
    ref, msg = EF._reference(p, 'add', key=('mixed', 'add', wide))
    EF.assert_matches(add0, p, 'add', ref, msg)
    EB.assert_grads_equal(g0, EB._reference(pb, ('mixed', precision, 'x')))
    lib_options(knob, value)
    _, _, add, mx, am, g = _neutral_run(precision)
    assert torch.equal(add, add0) and torch.equal(mx, mx0) and torch.equal(am, am0)
    for k in g0:
        assert torch.equal(g[k], g0[k]), k


# ---- 6. knobs a precision does not have, and pass counts without a shape ---------------------------------------------
def _launches_and_out(p, precision, aggr='add'):
    from graph_pde_b200 import nn_conv
    n0 = nn_conv.stats['launches']
    out, _ = EF._run(p, precision, aggr)
    return nn_conv.stats['launches'] - n0, out


@pytest.mark.gpu
@pytest.mark.parametrize('schedule', [s for s, (_, _, precs) in SCHEDULES.items() if 'f16x2' not in precs])
def test_per_batch_knobs_are_ignored_at_f16x2(schedule, lib_options, monkeypatch, formulation_c):
    """f16x2 has no per-batch kernels: under no_fuse (and the knobs of those kernels) it runs the fused kernel, with
    the default schedule's launches and bits, exactly."""
    p, wide = _mixed('f16x2')
    n_def, out_def = _launches_and_out(p, 'f16x2')
    _apply(schedule, 'f16x2', lib_options, monkeypatch)
    n, out = _launches_and_out(p, 'f16x2')
    assert n == n_def, (n, n_def)
    assert torch.equal(out, out_def)
    ref, msg = EF._reference(p, 'add', key=('mixed', 'add', wide))
    EF.assert_matches(out, p, 'add', ref, msg)


@pytest.mark.gpu
@pytest.mark.parametrize('precision', ALL)
def test_forced_pass_count_without_a_shape_is_ignored(precision, lib_options, formulation_c):
    """The mixed probe's Kp = 128 has 2 k-chunks (6 at f16x2, whose Y GEMM reads three of them per chunk): two passes
    would leave fewer than 4 B slots per pass.  apply_passes=2 then keeps the automatic shape: the fused kernel, with
    the default launches, at every precision.  (It used to make the shape unsupported: f16 and bf16 ran the per-batch
    kernels instead, and f16x2 was refused as a shape the tensor cores do not cover.)"""
    from graph_pde_b200 import _lib
    p, wide = _mixed(precision)
    n_def, out_def = _launches_and_out(p, precision)
    lib_options('apply_passes', 2)
    n, out = _launches_and_out(p, precision)
    assert n == n_def, (n, n_def)
    assert torch.equal(out, out_def)
    conv = p.conv(EF._cls(), precision, 'add', DEV)
    assert _lib.lib().nnconv_weights_tc_supported(conv._get_prepared(precision).handle) == 1
    ref, msg = EF._reference(p, 'add', key=('mixed', 'add', wide))
    EF.assert_matches(out, p, 'add', ref, msg)


@pytest.mark.gpu
@pytest.mark.parametrize('passes', [2, 3])
def test_forced_pass_counts_that_have_a_shape(passes, lib_options, monkeypatch, formulation_c):
    """hub_batches at f16x2: Kp = 256, so the fused kernel's K has 12 chunks and 2 or 3 forced passes leave 6 or 4 B
    slots per pass; add and mean, with the hub across ~100 flag batches."""
    lib_options('apply_passes', passes)
    _f_graph('hub_batches')('f16x2', {}, monkeypatch)


# ---- 7. the matrix can fail, where it should -------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('change', ['delete', 'duplicate', 'redirect'])
@pytest.mark.parametrize('aggr', ['add', 'mean'])
@pytest.mark.parametrize('schedule', ['scatter_mode0+ring2', 'per_batch_pdl'])
def test_one_changed_edge_fails_exactly_where_it_lands(schedule, aggr, change, lib_options, monkeypatch,
                                                       formulation_c):
    """test_gpu_exact_forward's sensitivity check under a fused and a per-batch schedule: one edge deleted, duplicated
    or sent to another target fails at exactly the nodes the change touched."""
    _apply(schedule, 'f16', lib_options, monkeypatch)
    EF.test_one_changed_edge_fails_exactly_where_it_lands(change, aggr)
