"""H100-native drop-in for the reference's edge-conditioned convolution.

Mirrors the operator interface of the reference (paths relative to neuraloperator/graph-pde):

* ``NNConv_old(in_channels, out_channels, nn, aggr='add', root_weight=True, bias=True, **kwargs)``
  -- graph-neural-operator/nn_conv.py:197-286 (ctor :234-259, reset_parameters :261-265,
  forward :267-271, message :273-275, update :277-282, __repr__ :284-286)
* ``NNConv`` -- the upstream ``torch_geometric.nn.NNConv`` imported by the MGKN scripts
  (multipole-graph-neural-operator/neurips1_MGKN.py:10,41; same math, same signature).

Same attribute names (``in_channels, out_channels, nn, aggr, root, bias``), same state-dict keys
(``nn.layers.{0,2,4}.{weight,bias}``, ``root``, ``bias``), same init distributions.  The arithmetic
runs in libnnconv_b200.so (hand-written sm_90a CUDA, C ABI in include/nnconv_b200.h); PyTorch only
owns the device memory and the stream.  There is no CPU / eager fallback: a CPU tensor, a missing
library or an unsupported edge network raises.

Algorithm (see DESIGN.md): the edge MLP minus its last Linear is x-independent, so its output
``h_e`` is computed once per (edge_attr, parameters) and cached across the T applications of the shared
conv in KernelNN.forward (graph-neural-operator/UAI1_full_resolution.py:29-30); each application then
runs ``m_e = h_e . Y_src + c_src`` with the per-source matrix ``Y_src = x_src (x) W_L`` and scatters
``m_e / deg`` into the target rows.
"""
import collections
import contextlib
import ctypes
import math
import os
import weakref

import torch
from torch.nn import Parameter

from . import _lib

__all__ = ['NNConv_old', 'NNConv', 'ECConv', 'DiagNNConv', 'stats', 'clear_caches', 'default_precision']

stats = {'launches': 0, 'plans_built': 0, 'edge_feature_passes': 0, 'edge_kernel_passes': 0, 'applies': 0,
         'weight_preps': 0, 'backwards': 0, 'mlp_backwards': 0, 'streamed_chunk_passes': 0,
         'streamed_backward_chunk_passes': 0}

_PLAN_CACHE = collections.OrderedDict()
_PLAN_CACHE_MAX = int(os.environ.get('NNCONV_B200_PLAN_CACHE', '64'))                 # entries
_PLAN_CACHE_MAX_BYTES = int(os.environ.get('NNCONV_B200_PLAN_CACHE_BYTES', str(2 << 30)))   # plan buffers + pinned edge_index
_OVERFLOW_CHECK = os.environ.get('NNCONV_B200_OVERFLOW_CHECK', '1') != '0'
_Y_BYTES = int(os.environ.get('NNCONV_B200_Y_BYTES', '0'))   # Y ring bytes; 0: the library sizes it from the device's L2
_EF_WS_BYTES = int(os.environ.get('NNCONV_B200_EF_WS_BYTES', str(2 << 30)))  # hidden-layer ping-pong chunk (fewer, larger chunks)
_BWD_WS_BYTES = int(os.environ.get('NNCONV_B200_BWD_WS_BYTES', str(2 << 30)))  # fp32 backward: activations per batch
# tensor-core backward: per-application workspace (dY of a source batch; larger = fewer batches) and the per-batch
# buffers of the deferred pass through the hidden layers.  Sized so that a 241^2 training step (47 GiB of edge features)
# fits an 80 GB H100.
_BWD_APPLY_WS_BYTES = int(os.environ.get('NNCONV_B200_BWD_APPLY_WS_BYTES', str(4 << 30)))
_BWD_MLP_WS_BYTES = int(os.environ.get('NNCONV_B200_BWD_MLP_WS_BYTES', str(4 << 30)))
_BWD_MODE = os.environ.get('NNCONV_B200_BACKWARD', 'auto')       # auto | tc | fp32
# training: keep the hidden activations h_1..h_{L-2} of the forward for the backward (2 KB per edge and layer at width
# 1024: 47 GiB at 241^2, which does not fit an 80 GB H100 beside the edge features) instead of recomputing them, when
# they fit this budget
_KEEP_ACTS_MAX_BYTES = int(os.environ.get('NNCONV_B200_KEEP_ACTS_BYTES', str(8 << 30)))
# per-edge kernel matrices (formulation B) for graphs with few out-edges per source: auto | on | off
_EDGE_KERNELS = os.environ.get('NNCONV_B200_EDGE_KERNELS', 'auto')
_EDGE_KERNELS_MAX_DEG = 8                       # auto: average out-degree of the sources with out-edges ...
# ... or a graph so small that streaming 8 KB per edge (<= 64 MB) costs less
_EDGE_KERNELS_MAX_EDGES = int(os.environ.get('NNCONV_B200_EDGE_KERNELS_MAX_EDGES', '8192'))
                                                # than the fixed cost of the persistent kernel (MGKN's coarse levels)
_EDGE_KERNELS_MAX_BYTES = 2 << 30
# budget (bytes) of the cached edge features h; a graph whose h is larger keeps a prefix of h resident and recomputes
# the rest chunk by chunk inside every application (see NNConv_old).  Unset: the whole h, streaming only on an OOM.
_EDGE_FEATURE_BYTES = os.environ.get('NNCONV_B200_EDGE_FEATURE_BYTES')
_STREAM_MARGIN_BYTES = 1 << 30     # left free beside the resident prefix when the budget comes from mem_get_info
# ... and in training, beside the backward's workspace: what else a step allocates (autograd's saved tensors, the
# backward thread's cuBLAS handle and workspace, optimizer state) and the caching allocator's fragmentation
_STREAM_TRAIN_MARGIN_BYTES = 4 << 30
# default of NNConv_old(streamed_training=...): '1' lets training run on streamed edge features (see NNConv_old)
_STREAMED_TRAINING = os.environ.get('NNCONV_B200_STREAMED_TRAINING', '0') == '1'
_MLP_GROUP = 6                     # applications per deferred pass through the hidden layers
# registered by capture.GraphedTrainStep while it captures a training step (see _CaptureSink), else None
_CAPTURE_SINK = None


def default_precision():
    return os.environ.get('NNCONV_B200_PRECISION', 'f16')


def clear_caches():
    _PLAN_CACHE.clear()
    from . import gcn          # the GCNConv graphs (gcn imports this module, so not at the top)
    gcn._GRAPH_CACHE.clear()


class _CaptureSink(object):
    """Where a CUDA-graph-captured training step reports fp16 overflow.  A captured pass cannot read its range counter
    on the host, so while this sink is registered every counter site enqueues nnconv_overflow_accumulate instead: the
    counter is added into ``words[0]``, and a K_e build's also into ``words[1]`` (the replay reads ``words[0]`` after
    the step and ``words[1]`` only to word its error).  ``plans`` keeps the plans the captured launches read alive for
    as long as the graph: an eviction from the plan cache would otherwise free buffers the graph still reads."""

    def __init__(self, device):
        self.words = torch.zeros(2, dtype=torch.int32, device=device)
        self.plans = {}


@contextlib.contextmanager
def _capturing_into(sink):
    global _CAPTURE_SINK
    _CAPTURE_SINK = sink
    try:
        yield sink
    finally:
        _CAPTURE_SINK = None


def _stream_ptr(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _f32(t):
    """``t`` detached, as the fp32 contiguous operand the library reads (None stays None: an absent root or bias).
    Already such a tensor, it is not converted: this runs several times per application on launch-bound graphs."""
    if t is None:
        return None
    t = t.detach()
    return t if t.dtype == torch.float32 and t.is_contiguous() else t.contiguous().float()


def _require_cuda(t, name):
    if not t.is_cuda:
        raise RuntimeError('graph_pde_b200.NNConv: `%s` must be a CUDA tensor (there is no CPU path); got %s'
                           % (name, t.device))


def _node_pair(n_nodes):
    """(N_src, N_dst) of a node count: an int N is the square graph (N, N), a pair a bipartite one."""
    if isinstance(n_nodes, (tuple, list)):
        return int(n_nodes[0]), int(n_nodes[1])
    return int(n_nodes), int(n_nodes)


def _in_pair(in_channels):
    """(in_src, in_dst) of ``in_channels``: an int means the same width on both sides."""
    if isinstance(in_channels, (tuple, list)):
        return int(in_channels[0]), int(in_channels[1])
    return in_channels, in_channels


def _node_sets(x, size, flow, in_dst):
    """(x, x_dst, N_dst) of a conv's ``x`` and ``size``, checked on the host before any launch.  A Tensor ``x`` is one
    node set: x_dst and N_dst are None, and a ``size`` must agree with its rows.  A pair ``(x_src, x_dst or None)`` is
    PyG's bipartite input (DESIGN 4.10): x = x_src, and x_dst must be [N_dst, in_dst]."""
    if not isinstance(x, (tuple, list)):
        x = x.unsqueeze(-1) if x.dim() == 1 else x
        if size is not None and any(n is not None and int(n) != x.size(0) for n in size):
            raise ValueError('size %s disagrees with x of %d rows (a Tensor x is one node set)'
                             % (tuple(size), x.size(0)))
        return x, None, None
    if len(x) != 2:
        raise ValueError('x must be a Tensor or a pair (x_src, x_dst), got a sequence of %d' % len(x))
    if flow != 'source_to_target':
        raise ValueError("a pair (x_src, x_dst) needs flow='source_to_target': under 'target_to_source' PyG takes "
                         'both the messages and the root term from x[1], which is not a bipartite map')
    x_src, x_dst = x
    x_src = x_src.unsqueeze(-1) if x_src.dim() == 1 else x_src
    if x_dst is not None:
        x_dst = x_dst.unsqueeze(-1) if x_dst.dim() == 1 else x_dst
    if size is not None:
        if len(size) != 2:
            raise ValueError('size must be (N_src, N_dst), got %s' % (tuple(size),))
        if size[0] is not None and int(size[0]) != x_src.size(0):
            raise ValueError('size[0] = %d disagrees with x_src of %d rows' % (int(size[0]), x_src.size(0)))
        if size[1] is not None and x_dst is not None and int(size[1]) != x_dst.size(0):
            raise ValueError('size[1] = %d disagrees with x_dst of %d rows' % (int(size[1]), x_dst.size(0)))
    if x_dst is not None:
        n_dst = x_dst.size(0)
    elif size is not None and size[1] is not None:
        n_dst = int(size[1])
    else:
        raise ValueError('x_dst = None needs size = (N_src, N_dst) to give the number of targets')
    if n_dst < 1:
        raise ValueError('a bipartite call needs at least one target, got N_dst = %d' % n_dst)
    if x_dst is not None:
        _require_cuda(x_dst, 'x_dst')
        if x_dst.dim() != 2 or x_dst.size(1) != in_dst:
            raise ValueError('x_dst has shape %s, expected [N_dst, %d]' % (tuple(x_dst.shape), in_dst))
    return x_src, x_dst, n_dst


class _Plan(object):
    """Per-edge_index preprocessing owned by the C library (nnconv_plan_t) + the buffers it lives in.  ``n_nodes``: N
    (square graph) or (N_src, N_dst) (bipartite: sources index x_src, targets the rows of out)."""

    def __init__(self, edge_index, n_nodes, flow):
        L = _lib.lib()
        _lib.check(L.nnconv_init())
        e = edge_index.size(1)
        n_src, n_dst = _node_pair(n_nodes)
        ws_b, tmp_b = ctypes.c_size_t(), ctypes.c_size_t()
        _lib.check(L.nnconv_plan_sizes_bipartite(e, n_src, n_dst, ctypes.byref(ws_b), ctypes.byref(tmp_b)))
        dev = edge_index.device
        self.ws = torch.empty(ws_b.value, dtype=torch.uint8, device=dev)
        tmp = torch.empty(tmp_b.value, dtype=torch.uint8, device=dev)
        row0, row1 = edge_index[0], edge_index[1]
        if row0.stride(0) != 1:
            row0 = row0.contiguous()
        if row1.stride(0) != 1:
            row1 = row1.contiguous()
        self._rows = (row0, row1)
        self.edge_index = edge_index          # keeps the storage (and so the cache key) alive
        h = ctypes.c_void_p()
        _lib.check(L.nnconv_plan_create_bipartite(_ptr(row0), _ptr(row1), e, n_src, n_dst, _lib.FLOW[flow],
                                                  _ptr(self.ws), ws_b.value, _ptr(tmp), tmp_b.value, _stream_ptr(dev),
                                                  ctypes.byref(h)))
        self.handle = h
        self.key = _plan_key(edge_index, n_nodes, flow)
        self.nbytes = self.ws.numel() + edge_index.numel() * edge_index.element_size()
        info = (ctypes.c_int64 * 8)()
        _lib.check(L.nnconv_plan_info(h, info, 8))
        self.E, self.N, self.n_src, self.n_tiles, self.max_out_deg, self.src_sorted = [int(v) for v in info[:6]]
        self.N_dst = int(info[7])        # rows of out (= N, the source count, on a square plan)
        stats['plans_built'] += 1
        self._finalizer = weakref.finalize(self, L.nnconv_plan_destroy, h)


class _EdgeFeatures(object):
    """The cached edge features of one (plan, prepared weights, edge_attr).  ``h`` holds the h of the sorted edges
    [0, E_res): the whole h when E_res = E, else a unit-aligned prefix, and every application recomputes the other
    edges' h in ``n_chunks`` chunks from ``ea32`` with a workspace of ``ws_bytes`` (nnconv_apply_streamed).  ``ea32``
    is also held so that its address cannot be recycled while it keys the cache.

    Beside h: the hidden activations kept for the tensor-core backward (``acts``, whole h only, else None); the
    formulation-B kernel matrices (``kmat``, built at the first application; ``kmat_overflow``: their build left the
    fp16 range, so formulation C computes these edges); the tensor-core backward's workspace when it was allocated with
    a prefix (``bwd_ws``, else None); and how a prefix was sized (``auto``: from the free device memory rather than a
    budget; ``for_grad``: leaving room for the backward)."""

    def __init__(self, h, E_res, E, n_chunks, ws_bytes, ea32, acts, bwd_ws, auto, for_grad):
        self.h, self.E_res, self.E, self.n_chunks, self.ws_bytes, self.ea32 = h, E_res, E, n_chunks, ws_bytes, ea32
        self.acts, self.bwd_ws, self.auto, self.for_grad = acts, bwd_ws, auto, for_grad
        self.kmat = None
        self.kmat_overflow = False

    @property
    def streamed(self):
        return self.E_res < self.E


def _streamed_chunks(plan, prepared, e_res, n_apps, ws_bytes):
    """Source batches whose edge features a streamed backward call recomputes (n_apps = 0: the per-application call)."""
    n = ctypes.c_int64(0)
    _lib.check(_lib.lib().nnconv_backward_streamed_chunks(plan.handle, prepared.handle, e_res, n_apps, ws_bytes,
                                                          ctypes.byref(n)))
    return n.value


def _plan_key(edge_index, n_nodes, flow):
    return (edge_index.data_ptr(), tuple(edge_index.shape), tuple(edge_index.stride()), edge_index._version,
            edge_index.device.index, _node_pair(n_nodes), flow)


def get_plan(edge_index, n_nodes, flow='source_to_target'):
    key = _plan_key(edge_index, n_nodes, flow)
    plan = _PLAN_CACHE.get(key)
    if plan is not None:
        _PLAN_CACHE.move_to_end(key)
        if _CAPTURE_SINK is not None:
            _CAPTURE_SINK.plans[key] = plan
        return plan
    plan = _Plan(edge_index, n_nodes, flow)
    _PLAN_CACHE[key] = plan
    # bounded by entries AND bytes (a 241^2 plan pins ~0.6 GB incl. the caller's edge_index); the newest plan stays
    while len(_PLAN_CACHE) > 1 and (len(_PLAN_CACHE) > _PLAN_CACHE_MAX or
                                    sum(p.nbytes for p in _PLAN_CACHE.values()) > _PLAN_CACHE_MAX_BYTES):
        _PLAN_CACHE.popitem(last=False)
    return plan


# hidden activations the library runs: each has a derivative that is a function of its output (include/nnconv_b200.h
# NNCONV_ACT_*), so the backward needs nothing beyond the activations it keeps for ReLU
_SELU_SCALE, _SELU_ALPHA = 1.0507009873554805, 1.6732632423543772    # torch.nn.SELU's constants


def _act_spec(m):
    """('relu' | 'leaky_relu' | 'elu' | 'tanh' | 'sigmoid', parameter) of an activation module, or for the kinds with
    a parameter block ('clamp' | 'scaled_elu' | 'softsign' | 'logsigmoid', tuple of parameters); None for any other
    module.  Raises NotImplementedError for an activation the library does not run, naming the reason.  Two specs are
    equal exactly when they are the same function: ReLU6() and Hardtanh(0, 6) are both ('clamp', (1, 0, 0, 6))."""
    if isinstance(m, torch.nn.ReLU):
        return ('relu', 0.0)
    if isinstance(m, torch.nn.LeakyReLU):
        if m.negative_slope < 0:
            raise NotImplementedError('edge network: LeakyReLU with a negative slope (%g) is not supported: its '
                                      'derivative is not a function of its output' % m.negative_slope)
        return ('leaky_relu', float(m.negative_slope))
    if isinstance(m, torch.nn.ELU):
        if m.alpha < 0:
            raise NotImplementedError('edge network: ELU with a negative alpha (%g) is not supported: its derivative '
                                      'is not a function of its output' % m.alpha)
        return ('elu', float(m.alpha))
    if isinstance(m, torch.nn.Tanh):
        return ('tanh', 0.0)
    if isinstance(m, torch.nn.Sigmoid):
        return ('sigmoid', 0.0)
    if isinstance(m, torch.nn.Hardtanh):           # ReLU6 is Hardtanh(0, 6); torch requires min_val < max_val
        return ('clamp', (1.0, 0.0, float(m.min_val), float(m.max_val)))
    if isinstance(m, torch.nn.Hardsigmoid):
        return ('clamp', (1.0 / 6.0, 0.5, 0.0, 1.0))
    if isinstance(m, torch.nn.SELU):
        return ('scaled_elu', (_SELU_SCALE, _SELU_ALPHA, 1.0))
    if isinstance(m, torch.nn.CELU):
        if not m.alpha > 0:
            raise NotImplementedError('edge network: CELU with alpha <= 0 (%g) is not supported: CELU divides by '
                                      'alpha, and its derivative is not a function of its output' % m.alpha)
        return ('scaled_elu', (1.0, float(m.alpha), 1.0 / float(m.alpha)))
    if isinstance(m, torch.nn.Softsign):
        return ('softsign', ())
    if isinstance(m, torch.nn.LogSigmoid):
        return ('logsigmoid', ())
    if isinstance(m, (torch.nn.GELU, torch.nn.SiLU, torch.nn.Softplus, torch.nn.Mish, torch.nn.Hardswish)):
        raise NotImplementedError('edge network: %s is not supported: its derivative is not a function of its '
                                  'output, so the backward would have to recompute the pre-activations'
                                  % type(m).__name__)
    if isinstance(m, torch.nn.modules.batchnorm._BatchNorm):
        raise NotImplementedError('edge network: normalize=True (%s between the layers) is not supported'
                                  % type(m).__name__)
    return None


def _edge_network(nn_module):
    """The edge network must be the reference's DenseNet shape (graph-neural-operator/utilities.py:201-227):
    Linear (act Linear)* with one hidden activation ``act`` in {ReLU, LeakyReLU(s >= 0), ELU(alpha >= 0), Tanh,
    Sigmoid, Hardtanh, ReLU6, Hardsigmoid, SELU, CELU(alpha > 0), Softsign, LogSigmoid} after every Linear but the last,
    no output nonlinearity and normalize=False.  Returns (the Linear layers, the activation spec (kind, parameter));
    a single Linear has the spec ('relu', 0.0), which it never uses."""
    if type(nn_module).__name__ == 'DenseNet_sin':
        raise NotImplementedError('edge network: DenseNet_sin (torch.sin between the layers) is not supported: the '
                                  'derivative of sin is not a function of its output')
    mods = [m for m in nn_module.modules() if len(list(m.children())) == 0]
    lin = []
    act = None
    expect_linear = True
    for m in mods:
        if isinstance(m, torch.nn.Linear):
            if not expect_linear:
                raise NotImplementedError('edge network: two Linear layers without an activation in between (an '
                                          'activation applied inside forward(), like torch.sin, is not supported)')
            if m.bias is None:
                raise NotImplementedError('edge network: Linear without bias is not supported')
            lin.append(m)
            expect_linear = False
            continue
        spec = _act_spec(m)
        if spec is None:
            raise NotImplementedError('edge network: only Linear chains with ReLU, LeakyReLU, ELU, Tanh, Sigmoid, '
                                      'Hardtanh, ReLU6, Hardsigmoid, SELU, CELU, Softsign or LogSigmoid between them '
                                      '(DenseNet) are supported, found %s' % type(m).__name__)
        if expect_linear:
            if lin:
                raise NotImplementedError('edge network: two activations in a row (%s after an activation)'
                                          % type(m).__name__)
            raise NotImplementedError('edge network: %s must follow a Linear layer' % type(m).__name__)
        if act is not None and act != spec:
            raise NotImplementedError('edge network: mixed activations (%s and %s): one activation must follow every '
                                      'hidden Linear, as DenseNet builds it' % (act, spec))
        act = spec
        expect_linear = True
    if not lin or expect_linear:
        raise NotImplementedError('edge network must end with a Linear layer (no output nonlinearity: '
                                  'out_nonlinearity is not supported)')
    return lin, act if act is not None else ('relu', 0.0)


def _linear_chain(nn_module):
    """The Linear layers of a ReLU edge network, Linear (ReLU Linear)*; any other edge network raises
    NotImplementedError.  The library's own code reads the network with _edge_network, which also accepts the other
    hidden activations."""
    lin, act = _edge_network(nn_module)
    if act[0] != 'relu':
        raise NotImplementedError('edge network: _linear_chain reads ReLU chains only, found %s' % (act,))
    return lin


def _act_params(act):
    """(float array, count) of an activation spec for nnconv_*weights_create_act_params: the tuple of a spec with a
    parameter block, the single parameter of the others."""
    p = act[1] if isinstance(act[1], tuple) else (act[1],)
    return (ctypes.c_float * max(len(p), 1))(*p), len(p)


class _Prepared(object):
    """nnconv_weights_t: padded / permuted / down-converted snapshot of the edge-MLP parameters."""

    def __init__(self, linears, cin, cout, precision, act=('relu', 0.0)):
        L = _lib.lib()
        _lib.check(L.nnconv_init())
        n = len(linears)
        dims = [linears[0].in_features] + [l.out_features for l in linears]
        c_dims = (ctypes.c_int * (n + 1))(*dims)
        nbytes = ctypes.c_size_t()
        prec = _lib.PREC[precision]
        _lib.check(L.nnconv_weights_sizes(n, c_dims, cin, cout, prec, ctypes.byref(nbytes)))
        dev = linears[0].weight.device
        self.buf = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        ws = [l.weight.detach().contiguous().float() for l in linears]
        bs = [l.bias.detach().contiguous().float() for l in linears]
        wp = (ctypes.c_void_p * n)(*[w.data_ptr() for w in ws])
        bp = (ctypes.c_void_p * n)(*[b.data_ptr() for b in bs])
        h = ctypes.c_void_p()
        q, nq = _act_params(act)
        _lib.check(L.nnconv_weights_create_act_params(n, c_dims, cin, cout, prec, _lib.ACT[act[0]], q, nq, wp, bp,
                                                      _ptr(self.buf), nbytes.value, _stream_ptr(dev), ctypes.byref(h)))
        self._keep = (ws, bs)
        self.handle = h
        self.dims = dims
        self.precision = precision
        self.act = act
        self.tc = bool(L.nnconv_weights_tc_supported(h))
        self.bwd_tc = bool(L.nnconv_backward_tc_supported(h))
        stats['weight_preps'] += 1
        stats['launches'] += 2 * n + 1
        self._finalizer = weakref.finalize(self, L.nnconv_weights_destroy, h)


class _NNConvFunction(torch.autograd.Function):
    """Differentiable wrapper, CUDA-core variant: forward = the configured precision path, backward =
    nnconv_backward_ex (fp32 CUDA-core kernels, csrc/backward.cu; any shape, activations recomputed).  Gradients flow
    to x, edge_attr, the edge-MLP Linear weights/biases, root and bias; edge_index gets none.  A bipartite call
    (``n_dst`` not None) takes x = x_src and the nullable x_dst, and its gradient also flows to x_dst."""

    @staticmethod
    def forward(ctx, module, x, edge_index, edge_attr, x_dst, n_dst, *params):
        ctx.module = module
        ctx.edge_index = edge_index
        ctx.pair = None if n_dst is None else _Pair(_f32(x_dst), n_dst)
        ctx.x_dst_dtype = x_dst.dtype if x_dst is not None else None
        ctx.save_for_backward(x, edge_attr)
        out, ctx.argmax = module._forward_impl(x, edge_index, edge_attr, for_grad=True, with_argmax=True, pair=ctx.pair)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        module = ctx.module
        x, edge_attr = ctx.saved_tensors
        grads = module._backward_impl(x, ctx.edge_index, edge_attr, grad_out, want_ea=ctx.needs_input_grad[3],
                                      argmax=ctx.argmax, pair=ctx.pair)
        # order of *params in forward(): list(module.parameters())
        by_id = {id(p): g for p, g in grads['params']}
        gxd = grads.get('x_dst')
        gxd = gxd.to(ctx.x_dst_dtype) if gxd is not None and ctx.needs_input_grad[4] else None
        return (None, grads['x'] if ctx.needs_input_grad[1] else None, None, grads.get('edge_attr'), gxd, None) + tuple(
            by_id.get(id(p)) for p in module.parameters())


class _Pair(object):
    """The target side of a bipartite call: x_dst (fp32, or None: no root term) and the target count N_dst."""

    def __init__(self, x_dst, n_dst):
        self.x_dst, self.n_dst = x_dst, n_dst


class _TrainState(object):
    """What the tensor-core backward shares between the applications of one conv on one (edge_attr, parameters):
    the plan, the prepared weights, the cached edge features (an _EdgeFeatures) and, filled during the backward sweep,
    every application's (grad_out, x, argmax) for the ONE deferred pass through the hidden layers (argmax: the
    forward's winning edges under aggr='max', else None)."""

    def __init__(self, key, plan, prepared, ef):
        self.key, self.plan, self.prepared, self.ef = key, plan, prepared, ef
        self.apps = []
        self.consumed = False
        self.token = None

    @property
    def acts(self):
        """The hidden activations the forward kept for the deferred pass (None: it recomputes them, or it has run)."""
        return self.ef.acts if self.ef is not None else None


class _EdgeFeaturesFn(torch.autograd.Function):
    """Autograd node of the x-independent part h = MLP_without_last_Linear(edge_attr).  Its output is a 1-element
    token (h itself lives in the module's cache: 2 KB per edge): every application's backward returns a dummy
    gradient for the token, so autograd runs THIS backward exactly once, after all of them -- with every
    (grad_out, x) pair collected in the state, the hidden layers are differentiated once for all T applications.
    edge_attr is an input so that its gradient (summed over the applications) comes out of the same pass."""

    @staticmethod
    def forward(ctx, module, state, edge_attr, *hidden_params):
        ctx.module, ctx.state = module, state
        ctx.ea_dtype = edge_attr.dtype
        return torch.zeros(1, device=edge_attr.device)

    @staticmethod
    def backward(ctx, _):
        state = ctx.state
        grads, gea = ctx.module._backward_mlp_impl(state, want_ea=ctx.needs_input_grad[2])
        state.consumed = True
        state.apps = []
        state.ef = None         # the per-edge buffers are no longer pinned by this (finished) graph
        return (None, None, gea.to(ctx.ea_dtype) if gea is not None else None) + tuple(grads)


class _ApplyFn(torch.autograd.Function):
    """One NNConv application given the edge features (tensor-core forward and backward).  A bipartite call (``n_dst``
    not None) takes x = x_src and the nullable x_dst; a square one passes None for both."""

    @staticmethod
    def forward(ctx, module, state, x, token, w_last, b_last, root, bias, x_dst, n_dst):
        ctx.module, ctx.state = module, state
        x32 = _f32(x)
        ctx.save_for_backward(x32)
        ctx.x_dtype = x.dtype
        ctx.pair = None if n_dst is None else _Pair(_f32(x_dst), n_dst)
        ctx.x_dst_dtype = x_dst.dtype if x_dst is not None else None
        out, ctx.argmax = module._apply_impl(state.plan, state.prepared, state.ef, x32, pair=ctx.pair)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        (x32,) = ctx.saved_tensors
        module, state = ctx.module, ctx.state
        g32 = _f32(grad_out)
        dx, dwl, dbl, droot, dbias, dxd = module._backward_apply_impl(state, x32, g32, ctx.argmax, ctx.pair)
        state.apps.append((g32, x32, ctx.argmax))
        dxd = dxd.to(ctx.x_dst_dtype) if dxd is not None and ctx.needs_input_grad[8] else None
        return (None, None, dx.to(ctx.x_dtype) if ctx.needs_input_grad[2] else None, torch.zeros_like(state.token),
                dwl, dbl, droot, dbias, dxd, None)


class NNConv_old(torch.nn.Module):
    r"""Edge-conditioned convolution  x'_i = Theta x_i + aggr_{j in N(i)} x_j . h_Theta(e_ij)
    (reference docstring: graph-neural-operator/nn_conv.py:198-232).

    Args are the reference's (nn_conv.py:234-241).  ``aggr`` in {'add', 'mean', 'max'}: 'max' takes the per-channel max
    of the messages (ties: the smallest index in the caller's edge_index; a node without in-edges gets 0) and sends each
    gradient entry to the winning edge only (DESIGN 5); it always runs formulation C.  Extra keyword ``precision`` in
    {'f16' (default), 'bf16', 'f16x2', 'fp32'} selects the tensor-core operand type: 'f16x2' carries every
    operand as an fp16 (hi, lo) pair -- fp32-grade results (tolerance 2e-5) on the tensor cores at ~2.4x the
    time of 'f16'; 'fp32' = CUDA-core path for arbitrary shapes.  ``flow`` is PyG's MessagePassing kwarg.

    ``edge_feature_bytes`` (default: environment NNCONV_B200_EDGE_FEATURE_BYTES, else unlimited) bounds the cached edge
    features (``Kp * 2`` bytes per edge, twice that at 'f16x2').  A graph whose features exceed it keeps a unit-aligned
    prefix resident and recomputes the rest chunk by chunk inside every application (same bits, more time); without a
    budget that happens only when allocating the whole h runs out of device memory.  Precision 'fp32' and the per-edge
    kernel matrices (graphs with few out-edges per source) never stream.

    ``streamed_training`` (default: environment NNCONV_B200_STREAMED_TRAINING == '1', else False) lets training run on
    such streamed features: the tensor-core backward recomputes the streamed part of h once per application and once
    more in the pass through the hidden layers (about 2T+1 edge-feature passes over the streamed edges per step instead
    of none), and the CUDA-core backward recomputes everything from edge_attr anyway.  Off, autograd through streamed
    features raises.  When the budget comes from the free device memory, the resident prefix leaves room for the
    backward's workspace.

    Bipartite input (PyG's form, DESIGN 4.10): ``in_channels`` may be a pair ``(in_src, in_dst)`` (an int means
    ``(in, in)``); the edge network then maps to ``in_src * out_channels``, ``root`` is ``[in_dst, out_channels]``, and
    ``reset_parameters`` draws root and bias from U(-1/sqrt(in_src), 1/sqrt(in_src)), the reference's rule applied to
    the message side.  ``forward(x, edge_index, edge_attr, size=None)`` accepts ``x = (x_src [N_src, in_src], x_dst
    [N_dst, in_dst] or None)``: ``out[i] = x_dst[i] root + bias + aggr_{e: dst_e = i} x_src[src_e] . nn(e)``, with
    N_dst rows; edge_index row 0 indexes x_src, row 1 x_dst.  ``x_dst = None`` drops the root term and needs ``size =
    (N_src, N_dst)``; a ``size`` that disagrees with the tensors raises ValueError, as do a pair under
    flow='target_to_source' and a pair passed to ``residual_step``.

    Caches: the down-converted weights and the x-independent edge features are cached per (parameter versions,
    edge_attr version).  Optimizer steps, ``load_state_dict`` and ``train()/eval()`` invalidate them; writes that
    bypass autograd's version counter (``p.data.copy_()``, ``p.data.clamp_()``) do NOT -- call ``invalidate()``
    after such writes.
    """

    def __init__(self, in_channels, out_channels, nn, aggr='add', root_weight=True, bias=True, **kwargs):
        super(NNConv_old, self).__init__()
        self.precision = kwargs.pop('precision', None)
        self.flow = kwargs.pop('flow', 'source_to_target')
        self.edge_feature_bytes = kwargs.pop('edge_feature_bytes', None)
        self.streamed_training = bool(kwargs.pop('streamed_training', _STREAMED_TRAINING))
        if kwargs:
            raise TypeError('unexpected keyword arguments %s' % sorted(kwargs))
        if aggr not in ('add', 'mean', 'max'):
            raise ValueError("aggr must be 'add', 'mean' or 'max'")
        if self.flow not in _lib.FLOW:
            raise ValueError('flow must be source_to_target or target_to_source')
        self.in_channels = tuple(in_channels) if isinstance(in_channels, (tuple, list)) else in_channels
        self.out_channels = out_channels
        self.nn = nn
        self.aggr = aggr
        if root_weight:
            self.root = Parameter(torch.Tensor(_in_pair(self.in_channels)[1], out_channels))
        else:
            self.register_parameter('root', None)
        if bias:
            self.bias = Parameter(torch.Tensor(out_channels))
        else:
            self.register_parameter('bias', None)
        self._prepared = {}             # slot ('forward' / 'backward') -> (key, _Prepared), see _get_prepared
        self._h_cache = {}              # at most one entry: cache key -> _EdgeFeatures
        self._tstate = None             # _TrainState of the tensor-core backward
        self._kmat_overflowed = set()   # plan keys whose K_e build left the fp16 range in an eager pass
        self.reset_parameters()

    # -- reference: nn_conv.py:261-265 with torch_geometric.nn.inits.reset / uniform restated ----------
    def reset_parameters(self):
        def _reset(m):
            children = list(m.children()) if hasattr(m, 'children') else []
            if children:
                for c in children:
                    _reset(c)
            elif hasattr(m, 'reset_parameters'):
                m.reset_parameters()
        _reset(self.nn)
        bound = 1.0 / math.sqrt(_in_pair(self.in_channels)[0])
        if self.root is not None:
            self.root.data.uniform_(-bound, bound)
        if self.bias is not None:
            self.bias.data.uniform_(-bound, bound)

    # -- reference: nn_conv.py:267-271 ------------------------------------------------------------------
    def forward(self, x, edge_index, edge_attr, size=None):
        pseudo = edge_attr.unsqueeze(-1) if edge_attr.dim() == 1 else edge_attr
        x, x_dst, n_dst = _node_sets(x, size, self.flow, _in_pair(self.in_channels)[1])
        nodes = x.size(0) if n_dst is None else (x.size(0), n_dst)
        needs_grad = torch.is_grad_enabled() and (
            x.requires_grad or pseudo.requires_grad or any(p.requires_grad for p in self.parameters()) or
            (x_dst is not None and x_dst.requires_grad))
        if needs_grad:
            state = self._train_state(x, edge_index, pseudo, nodes)
            if state is not None:            # tensor-core backward (csrc/backward_tc.cu)
                lin = _edge_network(self.nn)[0][-1]
                return _ApplyFn.apply(self, state, x, state.token, lin.weight, lin.bias, self.root, self.bias, x_dst,
                                      n_dst)
            return _NNConvFunction.apply(self, x, edge_index, pseudo, x_dst, n_dst, *list(self.parameters()))
        pair = None if n_dst is None else _Pair(_f32(x_dst), n_dst)
        return self._forward_impl(x, edge_index, pseudo, pair=pair)

    def __repr__(self):
        return '{}({}, {})'.format(self.__class__.__name__, self.in_channels, self.out_channels)

    # -- cache control ----------------------------------------------------------------------------------
    def invalidate(self):
        """Drop the prepared-weight snapshots and cached edge features (needed after parameter writes that do
        not bump the tensors' version counters, e.g. through ``.data``)."""
        self._prepared.clear()
        self._h_cache.clear()

    def train(self, mode=True):
        self.invalidate()
        return super(NNConv_old, self).train(mode)

    def _load_from_state_dict(self, *args, **kwargs):
        self.invalidate()
        return super(NNConv_old, self)._load_from_state_dict(*args, **kwargs)

    # -- host-side sequencing ---------------------------------------------------------------------------
    def _get_prepared(self, precision, slot='forward'):
        """Weight snapshot at ``precision``, cached per parameter versions in one of two slots: 'forward' (the
        edge-feature pass and the applications; a new snapshot drops the edge features of the old one) and 'backward'
        (the fp32 CUDA-core backward, whatever precision the forward runs at)."""
        linears, act = _edge_network(self.nn)
        key = (precision, act) + tuple((l.weight.data_ptr(), l.weight._version, l.bias.data_ptr(), l.bias._version)
                                       for l in linears)
        hit = self._prepared.get(slot)
        if hit is None or hit[0] != key:
            hit = self._prepared[slot] = (key, _Prepared(linears, _in_pair(self.in_channels)[0], self.out_channels,
                                                         precision, act))
            if slot == 'forward':
                self._h_cache.clear()
        return hit[1]

    def _budget(self):
        b = self.edge_feature_bytes
        if b is None and _EDGE_FEATURE_BYTES is not None:
            b = int(_EDGE_FEATURE_BYTES)
        return b

    def _streams(self, plan, prepared):
        """Whether these features may be streamed: 16-bit formulation C (the per-edge kernel matrices and fp32 need
        the whole h)."""
        return prepared.precision in ('f16', 'fp16', 'bf16', 'f16x2') and not self._wants_edge_kernels(plan, prepared)

    def edge_features(self, plan, prepared, edge_attr, keep_acts=False, for_grad=False):
        """x-independent part of message(), cached across the T applications of a shared conv: the buffer holding h of
        the resident edges (all of them unless the features stream; see _features)."""
        return self._features(plan, prepared, edge_attr, keep_acts, for_grad).h

    def _features(self, plan, prepared, edge_attr, keep_acts=False, for_grad=False):
        """The cached _EdgeFeatures of this call: the whole h or, when the whole h does not fit the budget or the
        device, a prefix of it (see the class docstring).  keep_acts: also keep the hidden activations for the
        backward (whole h only); for_grad: the features serve a training step."""
        key = (plan.key, edge_attr.data_ptr(), tuple(edge_attr.shape), edge_attr._version, id(prepared))
        L = _lib.lib()
        acts_b = ctypes.c_size_t(0)
        if keep_acts:
            _lib.check(L.nnconv_edge_acts_sizes(plan.handle, prepared.handle, ctypes.byref(acts_b)))
        acts_b = acts_b.value if acts_b.value <= _KEEP_ACTS_MAX_BYTES else 0
        hit = self._h_cache.get(key)
        if hit is not None:
            if hit.streamed:
                # a prefix keeps no activations.  Training may use it only with streamed_training (else the miss path
                # below raises), and not when it was sized from the free memory for inference: that prefix leaves no
                # room for the backward's workspace, so it is split again
                reuse = not for_grad or (self.streamed_training and (hit.for_grad or not hit.auto))
            else:
                reuse = not acts_b or hit.acts is not None
            if reuse:
                return hit
        h_b, ws_b = ctypes.c_size_t(), ctypes.c_size_t()
        _lib.check(L.nnconv_edge_features_sizes(plan.handle, prepared.handle, _EF_WS_BYTES, ctypes.byref(h_b),
                                                ctypes.byref(ws_b)))
        h_b, ws_b = h_b.value, ws_b.value
        dev = edge_attr.device
        self._h_cache.clear()                       # free the previous sample's features first
        budget = self._budget()
        streams = self._streams(plan, prepared)
        h = ws = acts = bwd_ws = None
        e_res, n_ch, chunk_ws_b = plan.E, 0, 0
        auto = False            # the prefix is sized from the free device memory: the whole h did not fit the device
        if budget is None or h_b <= budget or not streams:
            try:
                h = torch.empty(h_b, dtype=torch.uint8, device=dev)
                ws = torch.empty(ws_b, dtype=torch.uint8, device=dev)
            except torch.cuda.OutOfMemoryError:
                if not streams:
                    raise
                h = ws = None
                auto = True
        if h is None:
            if for_grad and not self.streamed_training:
                self._streaming_grad_error(h_b)
            if auto:
                self._tstate = None     # its reference to the previous h would hold memory the prefix is sized from

            def split(b):
                e, hb, cb, n = ctypes.c_int64(), ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_int64()
                _lib.check(L.nnconv_stream_split(plan.handle, prepared.handle, max(int(b), 0), _EF_WS_BYTES,
                                                 ctypes.byref(e), ctypes.byref(hb), ctypes.byref(cb), ctypes.byref(n)))
                return e.value, hb.value, cb.value, n.value

            e_res, h_res_b, chunk_ws_b, n_ch = split(0 if auto else budget)
            if auto:
                # the device's free memory only: the failed allocation above has already released the allocator's
                # unused segments, and what it still holds unallocated are free parts of segments in use -- fragments
                # that the 2 GiB workspaces below need not fit into
                free = torch.cuda.mem_get_info(dev)[0]
                work = chunk_ws_b + _STREAM_MARGIN_BYTES
                if for_grad:
                    # the streamed backward's workspaces do not depend on where the prefix ends: sized at E_res = 0
                    work += self._backward_reserve(plan, prepared, 0, edge_attr) + _STREAM_TRAIN_MARGIN_BYTES
                e_res, h_res_b, chunk_ws_b, n_ch = split(free - work)
            # training on the tensor cores: the backward's workspace (several GiB: 9 GiB at 241^2, f16x2) is allocated
            # here, beside the prefix, and reused by every backward call of this step.  Allocated per call, it would
            # need one contiguous block of that size after the forward has fragmented the caching allocator's segments.
            if for_grad and _BWD_MODE != 'fp32' and prepared.bwd_tc:
                # sized at E_res = 0: the streamed sizes do not depend on where the prefix ends, and they bound the
                # whole-h sizes should the prefix below end up covering every edge
                bwd_ws = torch.empty(self._tc_backward_ws_bytes(plan, prepared, 0), dtype=torch.uint8, device=dev)
            if e_res > 0:
                try:
                    h = torch.empty(h_res_b, dtype=torch.uint8, device=dev)
                except torch.cuda.OutOfMemoryError:
                    if not auto:
                        raise
                    e_res, h_res_b, chunk_ws_b, n_ch = split(0)
            if e_res > 0:
                ws = torch.empty(ws_b, dtype=torch.uint8, device=dev)
            else:
                h = torch.empty(0, dtype=torch.uint8, device=dev)     # every edge streams: no pass
        elif acts_b:
            acts = torch.empty(acts_b, dtype=torch.uint8, device=dev)
        if ws is not None:
            n_l = ctypes.c_int64(0)
            if acts is not None:
                _lib.check(L.nnconv_edge_features_keep(plan.handle, prepared.handle, _ptr(edge_attr), _ptr(h), _ptr(acts),
                                                       _ptr(ws), ws_b, _stream_ptr(dev), ctypes.byref(n_l)))
            else:
                _lib.check(L.nnconv_edge_features_prefix(plan.handle, prepared.handle, _ptr(edge_attr), e_res, _ptr(h),
                                                         _ptr(ws), ws_b, _stream_ptr(dev), ctypes.byref(n_l)))
            stats['launches'] += n_l.value
            stats['edge_feature_passes'] += 1
            self._check_overflow(prepared, ws, dev)
        ef = _EdgeFeatures(h, e_res, plan.E, n_ch, chunk_ws_b, edge_attr, acts, bwd_ws, auto, for_grad)
        self._h_cache[key] = ef
        return ef

    @staticmethod
    def _streaming_grad_error(nbytes):
        raise RuntimeError(
            'graph_pde_b200.NNConv: the edge features of this graph (%d bytes) do not fit on the device or in the cache '
            'budget, and training needs the whole h resident: streamed edge features are inference only (call '
            'under torch.no_grad(), or raise edge_feature_bytes / NNCONV_B200_EDGE_FEATURE_BYTES). Training on '
            'streamed edge features recomputes them in every backward application: enable it with '
            'streamed_training=True or NNCONV_B200_STREAMED_TRAINING=1' % nbytes)

    def _backward_reserve(self, plan, prepared, e_res, edge_attr):
        """Device bytes the backward of a training step on streamed features needs beside the resident prefix: its
        workspace plus the fp32 gradient w.r.t. edge_attr."""
        if _BWD_MODE != 'fp32' and prepared.bwd_tc:
            need = self._tc_backward_ws_bytes(plan, prepared, e_res)
        else:
            b = ctypes.c_size_t()
            _lib.check(_lib.lib().nnconv_backward_sizes(plan.handle, self._get_prepared('fp32', 'backward').handle,
                                                        _BWD_WS_BYTES, ctypes.byref(b)))
            need = b.value
        return need + 2 * edge_attr.numel() * 4

    @staticmethod
    def _tc_backward_ws_bytes(plan, prepared, e_res):
        """One workspace for the streamed tensor-core backward: its per-application calls and the MLP pass run one after
        the other on the stream, so the larger of the two sizes serves both."""
        L = _lib.lib()
        a, m = ctypes.c_size_t(), ctypes.c_size_t()
        _lib.check(L.nnconv_backward_apply_streamed_sizes(plan.handle, prepared.handle, e_res, _BWD_APPLY_WS_BYTES,
                                                          _EF_WS_BYTES, ctypes.byref(a)))
        _lib.check(L.nnconv_backward_mlp_streamed_sizes(plan.handle, prepared.handle, e_res, _MLP_GROUP,
                                                        _BWD_MLP_WS_BYTES, ctypes.byref(m)))
        return max(a.value, m.value)

    @staticmethod
    def _overflow_count(prepared, counter, dev, edge_kernels=False):
        """One host sync: the fp16 range counter at the start of ``counter`` (0 when the check is off, during CUDA-graph
        capture and for precisions without an fp16 range).  While a captured training step registers a _CaptureSink,
        the counter is added into the sink on the device instead (``edge_kernels``: a K_e build's counter)."""
        if not _OVERFLOW_CHECK or prepared.precision not in ('f16', 'fp16', 'f16x2'):
            return 0
        if torch.cuda.is_current_stream_capturing():
            sink = _CAPTURE_SINK
            if sink is not None:
                L = _lib.lib()
                for w in ((0, 1) if edge_kernels else (0,)):
                    _lib.check(L.nnconv_overflow_accumulate(_ptr(counter), ctypes.c_void_p(sink.words[w].data_ptr()),
                                                            _stream_ptr(dev)))
                    stats['launches'] += 1
            return 0
        cnt = ctypes.c_int64(0)
        _lib.check(_lib.lib().nnconv_edge_features_overflow(_ptr(counter), _stream_ptr(dev), ctypes.byref(cnt)))
        return cnt.value

    @staticmethod
    def _check_overflow(prepared, ws, dev):
        """One host sync: raise when edge-MLP activations written with ``ws`` left the fp16 range."""
        cnt = NNConv_old._overflow_count(prepared, ws, dev)
        if cnt:
            raise FloatingPointError(
                'graph_pde_b200.NNConv: %d blocks of edge-MLP activations left the fp16 range (|h| > 65504 or '
                "NaN); use precision='bf16' or 'fp32' for this parameter scale (NNCONV_B200_OVERFLOW_CHECK=0 "
                'disables this check and its one host sync per edge-feature pass)' % cnt)

    def _check_inputs(self, x, edge_index, pseudo):
        _require_cuda(x, 'x')
        _require_cuda(edge_index, 'edge_index')
        _require_cuda(pseudo, 'edge_attr')
        if edge_index.dtype != torch.int64 or edge_index.dim() != 2 or edge_index.size(0) != 2:
            raise ValueError('edge_index must be an int64 tensor of shape [2, E]')
        in_src = _in_pair(self.in_channels)[0]
        if x.size(1) != in_src:
            raise ValueError('x has %d channels, expected %d' % (x.size(1), in_src))
        if pseudo.size(0) != edge_index.size(1):
            raise ValueError('edge_attr has %d rows for %d edges' % (pseudo.size(0), edge_index.size(1)))

    def _prepare(self, x, edge_index, pseudo, keep_acts=False, for_grad=False, nodes=None):
        """plan, prepared weights, fp32 edge_attr and the (cached) edge features for this call; nodes: N_src or
        (N_src, N_dst), default x's rows."""
        precision = self.precision or default_precision()
        ea32 = _f32(pseudo)
        plan = get_plan(edge_index, x.size(0) if nodes is None else nodes, self.flow)
        prepared = self._get_prepared(precision)
        ef = self._features(plan, prepared, ea32, keep_acts and prepared.bwd_tc, for_grad)
        return plan, prepared, ea32, ef

    def _wants_edge_kernels(self, plan, prepared):
        """The graph-shape policy of formulation B (see _edge_kernels).  aggr='max' always runs formulation C."""
        if self.aggr == 'max' or _EDGE_KERNELS == 'off' or prepared.precision not in ('f16', 'fp16', 'bf16') or plan.E == 0:
            return False
        return _EDGE_KERNELS == 'on' or ((plan.E <= _EDGE_KERNELS_MAX_DEG * max(plan.n_src, 1) or
                                          plan.E <= _EDGE_KERNELS_MAX_EDGES) and
                                         plan.E * _in_pair(self.in_channels)[0] * self.out_channels * 2 <=
                                         _EDGE_KERNELS_MAX_BYTES)

    def _edge_kernels(self, plan, prepared, ef):
        """K_e = W_L h_e + b_L for every edge (formulation B) when the graph has few out-edges per source, else None.
        Kept with the edge features: as x-independent as they are."""
        if ef.streamed or ef.kmat_overflow or not self._wants_edge_kernels(plan, prepared):
            return None
        if ef.kmat is not None:
            return ef.kmat
        if _CAPTURE_SINK is not None and plan.key in self._kmat_overflowed:
            return None         # a captured step keeps the choice its eager warm-up made: formulation C
        L = _lib.lib()
        nbytes = ctypes.c_size_t()
        if L.nnconv_edge_kernels_sizes(plan.handle, prepared.handle, ctypes.byref(nbytes)) != _lib.OK:
            return None                                   # shape not covered: formulation C
        dev = ef.h.device
        kmat = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        _lib.check(L.nnconv_edge_kernels(plan.handle, prepared.handle, _ptr(ef.h), _ptr(kmat), _stream_ptr(dev)))
        stats['launches'] += 1
        stats['edge_kernel_passes'] += 1
        if self._overflow_count(prepared, kmat[nbytes.value - 1024:], dev, edge_kernels=True):
            # K_e left the fp16 range (it holds b_L in 16 bits): formulation C, which keeps b_L in fp32 and whose h and
            # Y passed their own checks, computes these edges instead
            ef.kmat_overflow = True
            self._kmat_overflowed.add(plan.key)
            return None
        ef.kmat = kmat
        return kmat

    def _apply_impl(self, plan, prepared, ef, x32, flags=0, pair=None):
        """One application: on the per-edge kernel matrices (formulation B, nnconv_apply_edge_ex), else on the whole h
        (nnconv_apply_ex), else on the resident prefix with the other edges' h recomputed in chunks
        (nnconv_apply_streamed: no allocation inside the library and, besides the optional overflow check, no host
        sync -- capturable by capture.GraphedForward).  aggr='max' takes nnconv_apply_max for either residency.
        Returns (out, argmax): argmax [N, out] int32 holds the winning caller edge of every (node, channel) under
        aggr='max' (-1: no in-edge), else None.  A bipartite call (pair: the _Pair of x_dst) runs the message part on
        x32 = x_src with no root or bias and then adds x_dst root + bias (nnconv_root_term); out has N_dst rows."""
        L = _lib.lib()
        dev = x32.device
        kmat = self._edge_kernels(plan, prepared, ef)
        keys_b = 0
        if kmat is None:
            ws_b = ctypes.c_size_t(ef.ws_bytes)         # a prefix: the size nnconv_stream_split gave it
            if not ef.streamed:
                _lib.check(L.nnconv_apply_sizes(plan.handle, prepared.handle, _Y_BYTES, ctypes.byref(ws_b)))
            if self.aggr == 'max':                      # the keys of the max precede the add / mean workspace
                max_b = ctypes.c_size_t()
                _lib.check(L.nnconv_apply_max_sizes(plan.handle, prepared.handle, ws_b.value, ctypes.byref(max_b)))
                keys_b = max_b.value - ws_b.value
                ws_b = max_b
            ws = torch.empty(ws_b.value, dtype=torch.uint8, device=dev)
        out = torch.empty(plan.N_dst, self.out_channels, dtype=torch.float32, device=dev)
        root, bias = (_f32(self.root), _f32(self.bias)) if pair is None else (None, None)
        aggr = _lib.AGGR[self.aggr]
        argmax = None
        if self.aggr == 'max':
            argmax = torch.empty(plan.N_dst, self.out_channels, dtype=torch.int32, device=dev)
            n_l = ctypes.c_int64(0)
            _lib.check(L.nnconv_apply_max(plan.handle, prepared.handle, _ptr(ef.ea32), _ptr(ef.h), ef.E_res, _ptr(x32),
                                          _ptr(root), _ptr(bias), flags, _ptr(out), _ptr(argmax), _ptr(ws), ws.numel(),
                                          _stream_ptr(dev), ctypes.byref(n_l)))
            stats['launches'] += n_l.value
        elif kmat is not None:
            _lib.check(L.nnconv_apply_edge_ex(plan.handle, prepared.handle, _ptr(kmat), _ptr(x32), _ptr(root), _ptr(bias),
                                              aggr, flags, _ptr(out), _stream_ptr(dev)))
            stats['launches'] += 2
        else:
            n_l = ctypes.c_int64(0)
            if ef.streamed:
                _lib.check(L.nnconv_apply_streamed(plan.handle, prepared.handle, _ptr(ef.ea32), _ptr(ef.h), ef.E_res,
                                                   _ptr(x32), _ptr(root), _ptr(bias), aggr, flags, _ptr(out), _ptr(ws),
                                                   ws.numel(), _stream_ptr(dev), ctypes.byref(n_l)))
            else:
                _lib.check(L.nnconv_apply_ex(plan.handle, prepared.handle, _ptr(ef.h), _ptr(x32), _ptr(root), _ptr(bias),
                                             aggr, flags, _ptr(out), _ptr(ws), ws.numel(), _stream_ptr(dev),
                                             ctypes.byref(n_l)))
            stats['launches'] += n_l.value
        if pair is not None:
            self._root_term(pair, out)
        stats['applies'] += 1
        if ef.n_chunks:
            stats['streamed_chunk_passes'] += ef.n_chunks
            self._check_overflow(prepared, ws[keys_b:], dev)    # its first word: fp16 overflows of the chunks
        return out, argmax

    def _root_term(self, pair, out):
        """out += x_dst root + bias of a bipartite call (no root term without x_dst)."""
        root = _f32(self.root) if pair.x_dst is not None else None
        bias = _f32(self.bias)
        if root is None and bias is None:
            return
        _lib.check(_lib.lib().nnconv_root_term(_ptr(pair.x_dst if root is not None else None), _ptr(root), _ptr(bias),
                                               out.size(0), _in_pair(self.in_channels)[1], self.out_channels, _ptr(out),
                                               _stream_ptr(out.device)))
        stats['launches'] += 1

    def _root_backward(self, pair, g32):
        """(grad x_dst or None, grad root or None, grad bias or None) of a bipartite call's root term."""
        dev = g32.device
        root = _f32(self.root) if pair.x_dst is not None else None
        dxd = torch.empty_like(pair.x_dst) if root is not None else None
        droot = torch.empty_like(self.root, dtype=torch.float32) if root is not None else None
        dbias = torch.empty_like(self.bias, dtype=torch.float32) if self.bias is not None else None
        if root is not None or dbias is not None:
            n_l = ctypes.c_int64(0)
            _lib.check(_lib.lib().nnconv_root_term_backward(
                _ptr(pair.x_dst if root is not None else None), _ptr(root), _ptr(g32), g32.size(0),
                _in_pair(self.in_channels)[1], self.out_channels, _ptr(dxd), _ptr(droot), _ptr(dbias),
                _stream_ptr(dev), ctypes.byref(n_l)))
            stats['launches'] += n_l.value
        if self.root is not None and droot is None:     # x_dst = None: root takes no part in the result
            droot = torch.zeros_like(self.root, dtype=torch.float32)
        return dxd, droot, dbias

    def _forward_impl(self, x, edge_index, pseudo, flags=0, for_grad=False, with_argmax=False, pair=None):
        """One application on the cached edge features; with_argmax: returns (out, argmax) (see _apply_impl)."""
        self._check_inputs(x, edge_index, pseudo)
        with torch.cuda.device(x.device):
            x32 = _f32(x)
            nodes = None if pair is None else (x32.size(0), pair.n_dst)
            plan, prepared, _, ef = self._prepare(x32, edge_index, pseudo, for_grad=for_grad, nodes=nodes)
            out, argmax = self._apply_impl(plan, prepared, ef, x32, flags, pair)
            return (out, argmax) if with_argmax else out

    def residual_step(self, z, edge_index, edge_attr, relu_in=True):
        """One V-cycle step ``x <- relu(x + conv(x))`` (multipole-graph-neural-operator/neurips1_MGKN.py:76,81,84) on
        PRE-activations, inference only: with ``x = relu(z)`` (``x = z`` if not ``relu_in``) returns
        ``z' = x + conv(x)``; the caller chains ``z'`` into the next step and applies the last ReLU itself.  The ReLU
        and the residual live in the node-prep launch of the application (``nnconv_apply_ex``), so a chain of steps
        has no elementwise kernels between its applications."""
        if isinstance(z, (tuple, list)):
            raise ValueError('residual_step needs one node set: x + conv(x) has no meaning for a pair (x_src, x_dst)')
        if _in_pair(self.in_channels) != (self.out_channels, self.out_channels):
            raise ValueError('residual_step needs in_channels == out_channels')
        if torch.is_grad_enabled() and (z.requires_grad or edge_attr.requires_grad or
                                        any(p.requires_grad for p in self.parameters())):
            raise RuntimeError('residual_step is a forward-only path: call it under torch.no_grad()')
        pseudo = edge_attr.unsqueeze(-1) if edge_attr.dim() == 1 else edge_attr
        flags = _lib.APPLY_RESIDUAL | (_lib.APPLY_RELU_IN if relu_in else 0)
        return self._forward_impl(z, edge_index, pseudo, flags)

    # -- tensor-core training path ----------------------------------------------------------------------
    def _train_state(self, x, edge_index, pseudo, nodes=None):
        """State shared by the applications of this conv on (edge_attr, parameters), or None when the tensor-core
        backward does not cover the configuration (the fp32 CUDA-core backward is used then)."""
        mode = _BWD_MODE
        if mode == 'fp32':
            return None
        self._check_inputs(x, edge_index, pseudo)
        with torch.cuda.device(x.device):
            plan, prepared, ea32, ef = self._prepare(x, edge_index, pseudo, keep_acts=True, for_grad=True, nodes=nodes)
            if not prepared.bwd_tc:
                if mode == 'tc':
                    raise NotImplementedError('NNCONV_B200_BACKWARD=tc: shape / precision not covered by the tensor-core backward')
                return None
            # requires_grad is part of the key: a state whose token is not connected to edge_attr cannot serve an
            # application that must deliver its gradient
            key = (plan.key, ea32.data_ptr(), tuple(ea32.shape), ea32._version, id(prepared), pseudo.requires_grad)
            st = self._tstate
            if st is None or st.key != key or st.consumed or st.ef is not ef:
                st = _TrainState(key, plan, prepared, ef)
                hidden = []
                for l in _edge_network(self.nn)[0][:-1]:
                    hidden += [l.weight, l.bias]
                st.token = _EdgeFeaturesFn.apply(self, st, pseudo, *hidden)
                self._tstate = st
            return st

    def _backward_apply_impl(self, state, x32, g32, argmax=None, pair=None):
        """Tensor-core backward of one application over the resident rows [0, E_res) of h; the other edges' h is
        recomputed per source batch.  With E_res = E this is the call nnconv_backward_apply makes.  argmax: the
        forward's, under aggr='max' (nnconv_backward_apply_max routes every gradient to its winning edge).  Returns
        (dx, dW_L, db_L, droot, dbias, dx_dst); a bipartite call (pair) takes droot, dbias and dx_dst from the root
        term's backward, else dx_dst is None."""
        L = _lib.lib()
        dev = x32.device
        plan, prep, ef = state.plan, state.prepared, state.ef
        lin = _edge_network(self.nn)[0][-1]
        with torch.cuda.device(dev):
            dx = torch.empty_like(x32)
            dwl = torch.empty_like(lin.weight, dtype=torch.float32)
            dbl = torch.empty_like(lin.bias, dtype=torch.float32)
            square = pair is None
            droot = torch.empty_like(self.root, dtype=torch.float32) if self.root is not None and square else None
            dbias = torch.empty_like(self.bias, dtype=torch.float32) if self.bias is not None and square else None
            root = _f32(self.root) if square else None
            ws = ef.bwd_ws
            if ws is None:
                b = ctypes.c_size_t()
                _lib.check(L.nnconv_backward_apply_streamed_sizes(plan.handle, prep.handle, ef.E_res, _BWD_APPLY_WS_BYTES,
                                                                  _EF_WS_BYTES, ctypes.byref(b)))
                ws = torch.empty(b.value, dtype=torch.uint8, device=dev)
            n_l = ctypes.c_int64(0)
            if self.aggr == 'max':
                _lib.check(L.nnconv_backward_apply_max(plan.handle, prep.handle, _ptr(ef.ea32), _ptr(ef.h), ef.E_res,
                                                       _ptr(x32), _ptr(root), _ptr(argmax), _ptr(g32), _ptr(dx), _ptr(dwl),
                                                       _ptr(dbl), _ptr(droot), _ptr(dbias), _ptr(ws), ws.numel(),
                                                       _stream_ptr(dev), ctypes.byref(n_l)))
            else:
                _lib.check(L.nnconv_backward_apply_streamed(plan.handle, prep.handle, _ptr(ef.ea32), _ptr(ef.h),
                                                            ef.E_res, _ptr(x32), _ptr(root), _lib.AGGR[self.aggr],
                                                            _ptr(g32), _ptr(dx), _ptr(dwl), _ptr(dbl), _ptr(droot),
                                                            _ptr(dbias), _ptr(ws), ws.numel(), _stream_ptr(dev),
                                                            ctypes.byref(n_l)))
            stats['launches'] += n_l.value
            if ef.streamed:
                stats['streamed_backward_chunk_passes'] += _streamed_chunks(plan, prep, ef.E_res, 0, ws.numel())
            dxd = None
            if not square:
                dxd, droot, dbias = self._root_backward(pair, g32)
            stats['backwards'] += 1
        return dx, dwl, dbl, droot, dbias, dxd

    def _backward_mlp_impl(self, state, want_ea=False):
        """Gradients of the hidden Linear layers, one pass for all applications recorded in the state (in groups
        of <= 6 when a conv is applied more often), and with ``want_ea`` the fp32 gradient w.r.t. edge_attr
        ([E, k_in], summed over the groups; else None)."""
        L = _lib.lib()
        plan, prep, ef = state.plan, state.prepared, state.ef
        hidden = _edge_network(self.nn)[0][:-1]
        dev = ef.ea32.device
        total = None
        gea_total = None
        with torch.cuda.device(dev):
            for i0 in range(0, len(state.apps), _MLP_GROUP):
                apps = state.apps[i0:i0 + _MLP_GROUP]
                n = len(apps)
                ws = ef.bwd_ws
                if ws is None:
                    b = ctypes.c_size_t()
                    _lib.check(L.nnconv_backward_mlp_streamed_sizes(plan.handle, prep.handle, ef.E_res, n,
                                                                    _BWD_MLP_WS_BYTES, ctypes.byref(b)))
                    ws = torch.empty(b.value, dtype=torch.uint8, device=dev)
                dws = [torch.empty_like(l.weight, dtype=torch.float32) for l in hidden]
                dbs = [torch.empty_like(l.bias, dtype=torch.float32) for l in hidden]
                gea = torch.empty(ef.ea32.shape, dtype=torch.float32, device=dev) if want_ea else None
                gp = (ctypes.c_void_p * n)(*[g.data_ptr() for g, _, _ in apps])
                xp = (ctypes.c_void_p * n)(*[x.data_ptr() for _, x, _ in apps])
                wp = (ctypes.c_void_p * len(hidden))(*[t.data_ptr() for t in dws])
                bp = (ctypes.c_void_p * len(hidden))(*[t.data_ptr() for t in dbs])
                if self.aggr == 'max':
                    # every application routed by its own forward's argmax
                    ap = (ctypes.c_void_p * n)(*[am.data_ptr() for _, _, am in apps])
                    _lib.check(L.nnconv_backward_mlp_max(plan.handle, prep.handle, _ptr(ef.ea32), _ptr(ef.h), ef.E_res, n,
                                                         gp, xp, ap, wp, bp, _ptr(ws), ws.numel(), _stream_ptr(dev),
                                                         _ptr(ef.acts), _ptr(gea)))
                elif ef.acts is not None:
                    _lib.check(L.nnconv_backward_mlp_ex(plan.handle, prep.handle, _ptr(ef.ea32), _ptr(ef.h), n, gp, xp,
                                                        _lib.AGGR[self.aggr], wp, bp, _ptr(ws), ws.numel(),
                                                        _stream_ptr(dev), _ptr(ef.acts), _ptr(gea)))
                else:
                    _lib.check(L.nnconv_backward_mlp_streamed(plan.handle, prep.handle, _ptr(ef.ea32), _ptr(ef.h),
                                                              ef.E_res, n, gp, xp, _lib.AGGR[self.aggr], wp, bp, _ptr(ws),
                                                              ws.numel(), _stream_ptr(dev), _ptr(gea)))
                if ef.streamed:
                    stats['streamed_backward_chunk_passes'] += _streamed_chunks(plan, prep, ef.E_res, n, ws.numel())
                flat = [t for pair in zip(dws, dbs) for t in pair]
                total = flat if total is None else [a + b for a, b in zip(total, flat)]
                if gea is not None:
                    gea_total = gea if gea_total is None else gea_total + gea
            stats['mlp_backwards'] += 1
        if total is None:     # no application contributed (cannot happen through autograd, kept for safety)
            total = [torch.zeros_like(p, dtype=torch.float32) for l in hidden for p in (l.weight, l.bias)]
            if want_ea:
                gea_total = torch.zeros(ef.ea32.shape, dtype=torch.float32, device=dev)
        return total, gea_total

    def _backward_impl(self, x, edge_index, pseudo, grad_out, want_ea=False, argmax=None, pair=None):
        """fp32 CUDA-core backward of one application; with ``want_ea`` also the gradient w.r.t. edge_attr
        (returned under 'edge_attr' in pseudo's dtype).  argmax: the forward's, under aggr='max' (whatever precision
        that forward ran at, the gradients follow its winning edges).  A bipartite call (pair) also returns the
        fp32 gradient w.r.t. x_dst under 'x_dst' (None without x_dst)."""
        L = _lib.lib()
        square = pair is None
        with torch.cuda.device(x.device):
            x32 = _f32(x)
            ea32 = _f32(pseudo)
            g32 = _f32(grad_out)
            n = x32.size(0)
            plan = get_plan(edge_index, n if square else (n, pair.n_dst), self.flow)
            linears = _edge_network(self.nn)[0]
            prep = self._get_prepared('fp32', 'backward')
            ws_b = ctypes.c_size_t()
            _lib.check(L.nnconv_backward_sizes(plan.handle, prep.handle, _BWD_WS_BYTES, ctypes.byref(ws_b)))
            ws = torch.empty(ws_b.value, dtype=torch.uint8, device=x.device)
            dx = torch.empty_like(x32)
            dws = [torch.empty_like(l.weight, dtype=torch.float32) for l in linears]
            dbs = [torch.empty_like(l.bias, dtype=torch.float32) for l in linears]
            droot = torch.empty_like(self.root, dtype=torch.float32) if self.root is not None and square else None
            dbias = torch.empty_like(self.bias, dtype=torch.float32) if self.bias is not None and square else None
            nl = len(linears)
            wp = (ctypes.c_void_p * nl)(*[t.data_ptr() for t in dws])
            bp = (ctypes.c_void_p * nl)(*[t.data_ptr() for t in dbs])
            root = _f32(self.root) if square else None
            gea = torch.empty_like(ea32) if want_ea else None
            if self.aggr == 'max':
                _lib.check(L.nnconv_backward_max(plan.handle, prep.handle, _ptr(ea32), _ptr(x32), _ptr(root), _ptr(argmax),
                                                 _ptr(g32), _ptr(dx), wp, bp, _ptr(droot), _ptr(dbias), _ptr(ws),
                                                 ws_b.value, _stream_ptr(x.device), _ptr(gea)))
            else:
                _lib.check(L.nnconv_backward_ex(plan.handle, prep.handle, _ptr(ea32), _ptr(x32), _ptr(root),
                                                _lib.AGGR[self.aggr], _ptr(g32), _ptr(dx), wp, bp, _ptr(droot),
                                                _ptr(dbias), _ptr(ws), ws_b.value, _stream_ptr(x.device), _ptr(gea)))
            dxd = None
            if not square:
                dxd, droot, dbias = self._root_backward(pair, g32)
            stats['backwards'] += 1
        params = [(l.weight, dw) for l, dw in zip(linears, dws)] + [(l.bias, db) for l, db in zip(linears, dbs)]
        if self.root is not None:
            params.append((self.root, droot))
        if self.bias is not None:
            params.append((self.bias, dbias))
        grads = {'x': dx.to(x.dtype), 'params': params, 'x_dst': dxd}
        if gea is not None:
            grads['edge_attr'] = gea.to(pseudo.dtype)
        return grads


class NNConv(NNConv_old):
    """Drop-in for upstream ``torch_geometric.nn.NNConv`` as the MGKN scripts use it
    (multipole-graph-neural-operator/neurips1_MGKN.py:41,49,57; MGKN_general_darcy2d.py:45,53,61;
    MGKN_orthogonal_burgers1d.py:37).  graph-neural-operator/nn_conv.py:8-96 also defines a class called NNConv, the
    diagonal-kernel variant: that one is DiagNNConv (and ``nn_conv.NNConv`` of the drop-in directory)."""
    pass


ECConv = NNConv


def _require_int_channels(conv, in_channels, out_channels):
    """The channel-wise convs (DiagNNConv, GaussianNNConv) have one width on both sides of a bipartite map: a pair
    ``in_channels`` raises NotImplementedError, as a non-square shape does."""
    if isinstance(in_channels, (tuple, list)):
        raise NotImplementedError(
            '%s: the channel-wise kernel needs one width C = in_channels = out_channels for x_src, x_dst and the output; '
            'got in_channels %s, out_channels %d' % (type(conv).__name__, tuple(in_channels), out_channels))


# ---------------------------------------------------------------------------------------------------------------------
# diagonal-kernel conv (formulation D, DESIGN 4.7)
# ---------------------------------------------------------------------------------------------------------------------
_DIAG_WS_BYTES = 1 << 30         # edge-network chunk of the d build (h rows + hidden activations)


class _DiagWeights(object):
    """nnconv_diag_weights_t: padded / down-converted snapshot of the edge network of a DiagNNConv."""

    def __init__(self, linears, channels, precision, act=('relu', 0.0)):
        L = _lib.lib()
        _lib.check(L.nnconv_init())
        n = len(linears)
        dims = [linears[0].in_features] + [l.out_features for l in linears]
        c_dims = (ctypes.c_int * (n + 1))(*dims)
        nbytes = ctypes.c_size_t()
        prec = _lib.PREC[precision]
        _lib.check(L.nnconv_diag_weights_sizes(n, c_dims, channels, prec, ctypes.byref(nbytes)))
        dev = linears[0].weight.device
        self.buf = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        ws = [l.weight.detach().contiguous().float() for l in linears]
        bs = [l.bias.detach().contiguous().float() for l in linears]
        wp = (ctypes.c_void_p * n)(*[w.data_ptr() for w in ws])
        bp = (ctypes.c_void_p * n)(*[b.data_ptr() for b in bs])
        h = ctypes.c_void_p()
        q, nq = _act_params(act)
        _lib.check(L.nnconv_diag_weights_create_act_params(n, c_dims, channels, prec, _lib.ACT[act[0]], q, nq, wp,
                                                           bp, _ptr(self.buf), nbytes.value, _stream_ptr(dev),
                                                           ctypes.byref(h)))
        self._keep = (ws, bs)
        self.handle = h
        self.precision = precision
        stats['weight_preps'] += 1
        self._finalizer = weakref.finalize(self, L.nnconv_diag_weights_destroy, h)


class _DiagFeatures(object):
    """d = W_L h + b_L of one (plan, weights, edge_attr): fp32 [E, out] in the plan's sorted edge order.  ``ea32`` is
    held so that its address cannot be recycled while it keys the cache."""

    def __init__(self, d, ea32):
        self.d, self.ea32 = d, ea32


class _DiagState(object):
    """What the applications of one DiagNNConv on one (edge_attr, parameters) share in training: the plan, d, and, when
    a gradient reaches the edge network (``for_mlp``), grad_d [E, out], into which every application's backward adds
    x_src * G_e before the ONE pass through the edge network (_DiagMlpFn, whose output is ``token``).  Without it dd and
    token stay None and the backward computes only the gradients of x, root and bias."""

    def __init__(self, key, plan, feats, out_channels, for_mlp):
        self.key, self.plan, self.feats = key, plan, feats
        self.dd = (torch.zeros(max(plan.E, 1), out_channels, dtype=torch.float32, device=feats.ea32.device)
                   if for_mlp else None)
        self.consumed = False
        self.token = None


class _DiagMlpFn(torch.autograd.Function):
    """Autograd node of d = nn(edge_attr): a 1-element token stands for d (which lives in the module's cache); every
    application returns a dummy gradient for it, so this backward runs once, after all of them, on their summed
    grad_d."""

    @staticmethod
    def forward(ctx, module, state, edge_attr, *mlp_params):
        ctx.module, ctx.state = module, state
        ctx.ea_dtype = edge_attr.dtype
        return torch.zeros(1, device=edge_attr.device)

    @staticmethod
    def backward(ctx, _):
        state = ctx.state
        grads, gea = ctx.module._backward_mlp_impl(state, want_ea=ctx.needs_input_grad[2])
        state.consumed = True
        state.dd = None
        return (None, None, gea.to(ctx.ea_dtype) if gea is not None else None) + tuple(grads)


class _DiagApplyFn(torch.autograd.Function):
    """One DiagNNConv application given d.  A bipartite call (``n_dst`` not None) takes x = x_src and the nullable
    x_dst; a square one passes None for both."""

    @staticmethod
    def forward(ctx, module, state, x, token, root, bias, x_dst, n_dst):
        ctx.module, ctx.state = module, state
        x32 = _f32(x)
        ctx.save_for_backward(x32)
        ctx.x_dtype = x.dtype
        ctx.pair = None if n_dst is None else _Pair(_f32(x_dst), n_dst)
        ctx.x_dst_dtype = x_dst.dtype if x_dst is not None else None
        out, ctx.argmax = module._apply_impl(state.plan, state.feats, x32, ctx.pair)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        (x32,) = ctx.saved_tensors
        state = ctx.state
        dx, droot, dbias, dxd = ctx.module._backward_apply_impl(state, x32, _f32(grad_out), ctx.argmax, ctx.pair)
        dxd = dxd.to(ctx.x_dst_dtype) if dxd is not None and ctx.needs_input_grad[6] else None
        return (None, None, dx.to(ctx.x_dtype) if ctx.needs_input_grad[2] else None,
                torch.zeros_like(state.token) if state.token is not None else None, droot, dbias, dxd, None)


class DiagNNConv(torch.nn.Module):
    r"""The diagonal-kernel edge-conditioned convolution of graph-neural-operator/nn_conv.py:8-96 (class ``NNConv``
    there):  x'_i = x_i root + bias + aggr_{j in N(i)} x_j * nn(e_ij), channel by channel.

    Same signature, attributes, state-dict keys and initialisation as NNConv_old (reference :47-73): the edge network
    ``nn`` is a Linear (act Linear)* chain (act: ReLU, LeakyReLU, ELU, Tanh or Sigmoid, see _edge_network) whose output
    width is ``out_channels``.  The reference multiplies x_j by
    ``diag_embed(nn(e)).view(-1, in, out)``, which is the diagonal matrix only when nn's output width, in_channels and
    out_channels are equal; any other shape raises NotImplementedError.  ``aggr`` in {'add', 'mean', 'max'} ('max':
    the rules of NNConv_old), ``precision`` in {'f16' (default), 'bf16', 'f16x2', 'fp32'} selects the edge network's
    operand type, ``flow`` is PyG's MessagePassing kwarg.

    d_e = nn(e) is x-independent: it is computed once per (edge_attr, parameters), chunk by chunk so that the hidden
    activations of the edge network are never held for the whole graph, and kept in fp32 (4 * out bytes per edge).
    Each application is one pass over d.  The backward computes every gradient on the CUDA cores in fp32, recomputing
    the edge network's activations from edge_attr once per backward pass for all applications of a shared conv.  Cache
    rules are NNConv_old's: ``invalidate()`` after parameter writes that bypass autograd's version counter.

    Bipartite input (PyG's form, DESIGN 4.10): ``forward(x, edge_index, edge_attr, size=None)`` also accepts ``x =
    (x_src [N_src, C], x_dst [N_dst, C] or None)`` and returns ``out[i] = x_dst[i] root + bias + aggr_{e: dst_e = i}
    x_src[src_e] * nn(e)`` over N_dst rows, with NNConv_old's rules for ``size``, ``x_dst = None``, the aggregations and
    the refusals.  ``in_channels`` stays an int: the diagonal kernel has one width C on both sides, and a pair raises
    NotImplementedError.
    """

    def __init__(self, in_channels, out_channels, nn, aggr='add', root_weight=True, bias=True, **kwargs):
        super(DiagNNConv, self).__init__()
        self.precision = kwargs.pop('precision', None)
        self.flow = kwargs.pop('flow', 'source_to_target')
        if kwargs:
            raise TypeError('unexpected keyword arguments %s' % sorted(kwargs))
        if aggr not in ('add', 'mean', 'max'):
            raise ValueError("aggr must be 'add', 'mean' or 'max'")
        if self.flow not in _lib.FLOW:
            raise ValueError('flow must be source_to_target or target_to_source')
        _require_int_channels(self, in_channels, out_channels)
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.nn = nn
        self.aggr = aggr
        if root_weight:
            self.root = Parameter(torch.Tensor(in_channels, out_channels))
        else:
            self.register_parameter('root', None)
        if bias:
            self.bias = Parameter(torch.Tensor(out_channels))
        else:
            self.register_parameter('bias', None)
        self._prepared = {}             # slot ('forward' / 'backward') -> (key, _DiagWeights)
        self._d_cache = {}              # at most one entry: cache key -> _DiagFeatures
        self._tstate = None             # _DiagState of the current training step
        self.reset_parameters()

    reset_parameters = NNConv_old.reset_parameters
    __repr__ = NNConv_old.__repr__
    _root_term = NNConv_old._root_term
    _root_backward = NNConv_old._root_backward

    def invalidate(self):
        """Drop the prepared-weight snapshots and the cached d."""
        self._prepared.clear()
        self._d_cache.clear()

    def train(self, mode=True):
        self.invalidate()
        return super(DiagNNConv, self).train(mode)

    def _load_from_state_dict(self, *args, **kwargs):
        self.invalidate()
        return super(DiagNNConv, self)._load_from_state_dict(*args, **kwargs)

    def _check_shape(self):
        lin = _edge_network(self.nn)[0]
        k = lin[-1].out_features
        if not (k == self.in_channels == self.out_channels):
            raise NotImplementedError(
                'DiagNNConv: the diagonal kernel needs nn output width == in_channels == out_channels; got nn output '
                '%d, in_channels %d, out_channels %d' % (k, self.in_channels, self.out_channels))
        return lin

    # -- reference: nn_conv.py:79-84 -----------------------------------------------------------------------------
    def forward(self, x, edge_index, edge_attr, size=None):
        x, x_dst, n_dst = _node_sets(x, size, self.flow, self.in_channels)
        pseudo = edge_attr.unsqueeze(-1) if edge_attr.dim() == 1 else edge_attr
        lin = self._check_shape()
        NNConv_old._check_inputs(self, x, edge_index, pseudo)
        needs_grad = torch.is_grad_enabled() and (
            x.requires_grad or pseudo.requires_grad or any(p.requires_grad for p in self.parameters()) or
            (x_dst is not None and x_dst.requires_grad))
        with torch.cuda.device(x.device):
            plan = get_plan(edge_index, x.size(0) if n_dst is None else (x.size(0), n_dst), self.flow)
            ea32 = _f32(pseudo)
            feats = self._features(plan, ea32)
            if not needs_grad:
                pair = None if n_dst is None else _Pair(_f32(x_dst), n_dst)
                return self._apply_impl(plan, feats, _f32(x), pair)[0]
            params = [t for l in lin for t in (l.weight, l.bias)]
            for_mlp = pseudo.requires_grad or any(p.requires_grad for p in params)
            key = (plan.key, ea32.data_ptr(), tuple(ea32.shape), ea32._version, id(feats), pseudo.requires_grad, for_mlp)
            st = self._tstate
            if st is None or st.key != key or st.consumed:
                st = _DiagState(key, plan, feats, self.out_channels, for_mlp)
                if for_mlp:
                    st.token = _DiagMlpFn.apply(self, st, pseudo, *params)
                self._tstate = st
            return _DiagApplyFn.apply(self, st, x, st.token, self.root, self.bias, x_dst, n_dst)

    # -- host-side sequencing ------------------------------------------------------------------------------------
    def _get_prepared(self, precision, slot='forward'):
        linears, act = _edge_network(self.nn)
        key = (precision, act) + tuple((l.weight.data_ptr(), l.weight._version, l.bias.data_ptr(), l.bias._version)
                                       for l in linears)
        hit = self._prepared.get(slot)
        if hit is None or hit[0] != key:
            hit = self._prepared[slot] = (key, _DiagWeights(linears, self.out_channels, precision, act))
            if slot == 'forward':
                self._d_cache.clear()
        return hit[1]

    def _features(self, plan, ea32):
        """The cached d of this (plan, parameters, edge_attr), built by nnconv_diag_build on a miss."""
        prepared = self._get_prepared(self.precision or default_precision())
        key = (plan.key, ea32.data_ptr(), tuple(ea32.shape), ea32._version, id(prepared))
        hit = self._d_cache.get(key)
        if hit is not None:
            return hit
        self._d_cache.clear()
        L = _lib.lib()
        d_b, ws_b = ctypes.c_size_t(), ctypes.c_size_t()
        _lib.check(L.nnconv_diag_sizes(plan.handle, prepared.handle, _DIAG_WS_BYTES, ctypes.byref(d_b), ctypes.byref(ws_b)))
        dev = ea32.device
        d = torch.empty(d_b.value // 4, dtype=torch.float32, device=dev)
        ws = torch.empty(ws_b.value, dtype=torch.uint8, device=dev)
        n_l = ctypes.c_int64(0)
        _lib.check(L.nnconv_diag_build(plan.handle, prepared.handle, _ptr(ea32), _ptr(d), _ptr(ws), ws_b.value,
                                       _stream_ptr(dev), ctypes.byref(n_l)))
        stats['launches'] += n_l.value
        stats['edge_feature_passes'] += 1
        NNConv_old._check_overflow(prepared, ws, dev)
        feats = _DiagFeatures(d, ea32)
        feats.prepared = prepared
        self._d_cache[key] = feats
        return feats

    def _apply_impl(self, plan, feats, x32, pair=None):
        """One application (nnconv_apply_diag); returns (out, argmax), argmax None unless aggr='max'.  A bipartite call
        (pair: the _Pair of x_dst) runs the messages from x32 = x_src with no root or bias, then adds x_dst root + bias
        (nnconv_root_term); out has N_dst rows."""
        L = _lib.lib()
        dev = x32.device
        aggr = _lib.AGGR[self.aggr]
        ws_b = ctypes.c_size_t()
        _lib.check(L.nnconv_apply_diag_sizes(plan.handle, feats.prepared.handle, aggr, ctypes.byref(ws_b)))
        ws = torch.empty(ws_b.value, dtype=torch.uint8, device=dev)
        out = torch.empty(plan.N_dst, self.out_channels, dtype=torch.float32, device=dev)
        argmax = torch.empty(plan.N_dst, self.out_channels, dtype=torch.int32, device=dev) if self.aggr == 'max' else None
        root, bias = (_f32(self.root), _f32(self.bias)) if pair is None else (None, None)
        n_l = ctypes.c_int64(0)
        _lib.check(L.nnconv_apply_diag(plan.handle, feats.prepared.handle, _ptr(feats.d), _ptr(x32), _ptr(root),
                                       _ptr(bias), aggr, _ptr(out), _ptr(argmax), _ptr(ws), ws_b.value,
                                       _stream_ptr(dev), ctypes.byref(n_l)))
        stats['launches'] += n_l.value
        if pair is not None:
            self._root_term(pair, out)
        stats['applies'] += 1
        return out, argmax

    def _backward_apply_impl(self, state, x32, g32, argmax, pair=None):
        """dx, droot, dbias, dx_dst of one application; adds its share into state.dd (when the edge network needs it).
        A bipartite call (pair) takes droot, dbias and dx_dst from the root term's backward, else dx_dst is None."""
        L = _lib.lib()
        dev = x32.device
        with torch.cuda.device(dev):
            square = pair is None
            dx = torch.empty_like(x32)
            droot = torch.empty_like(self.root, dtype=torch.float32) if self.root is not None and square else None
            dbias = torch.empty_like(self.bias, dtype=torch.float32) if self.bias is not None and square else None
            root = _f32(self.root) if square else None
            n_l = ctypes.c_int64(0)
            _lib.check(L.nnconv_backward_apply_diag(state.plan.handle, state.feats.prepared.handle, _ptr(state.feats.d),
                                                    _ptr(x32), _ptr(root), _lib.AGGR[self.aggr], _ptr(argmax),
                                                    _ptr(g32), _ptr(dx), _ptr(droot), _ptr(dbias), _ptr(state.dd),
                                                    _stream_ptr(dev), ctypes.byref(n_l)))
            stats['launches'] += n_l.value
            dxd = None
            if not square:
                dxd, droot, dbias = self._root_backward(pair, g32)
            stats['backwards'] += 1
        return dx, droot, dbias, dxd

    def _backward_mlp_impl(self, state, want_ea=False):
        """Gradients of every Linear of the edge network (weight, bias, in order) from the summed grad_d, and with
        ``want_ea`` the fp32 gradient w.r.t. edge_attr."""
        L = _lib.lib()
        ea32 = state.feats.ea32
        dev = ea32.device
        linears = _edge_network(self.nn)[0]
        with torch.cuda.device(dev):
            prep = self._get_prepared('fp32', 'backward')
            ws_b = ctypes.c_size_t()
            _lib.check(L.nnconv_backward_mlp_diag_sizes(state.plan.handle, prep.handle, _BWD_WS_BYTES, ctypes.byref(ws_b)))
            ws = torch.empty(ws_b.value, dtype=torch.uint8, device=dev)
            dws = [torch.empty_like(l.weight, dtype=torch.float32) for l in linears]
            dbs = [torch.empty_like(l.bias, dtype=torch.float32) for l in linears]
            gea = torch.empty_like(ea32) if want_ea else None
            wp = (ctypes.c_void_p * len(linears))(*[t.data_ptr() for t in dws])
            bp = (ctypes.c_void_p * len(linears))(*[t.data_ptr() for t in dbs])
            _lib.check(L.nnconv_backward_mlp_diag(state.plan.handle, prep.handle, _ptr(ea32), _ptr(state.dd), wp, bp,
                                                  _ptr(ws), ws_b.value, _stream_ptr(dev), _ptr(gea)))
            stats['mlp_backwards'] += 1
        return [t for pair in zip(dws, dbs) for t in pair], gea
