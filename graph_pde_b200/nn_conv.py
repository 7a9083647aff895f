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

__all__ = ['NNConv_old', 'NNConv', 'ECConv', 'stats', 'clear_caches', 'default_precision']

stats = {'launches': 0, 'plans_built': 0, 'edge_feature_passes': 0, 'applies': 0, 'weight_preps': 0,
         'streamed_chunk_passes': 0, 'streamed_backward_chunk_passes': 0}

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


def _require_cuda(t, name):
    if not t.is_cuda:
        raise RuntimeError('graph_pde_b200.NNConv: `%s` must be a CUDA tensor (there is no CPU path); got %s'
                           % (name, t.device))


class _Plan(object):
    """Per-edge_index preprocessing owned by the C library (nnconv_plan_t) + the buffers it lives in."""

    def __init__(self, edge_index, n_nodes, flow):
        L = _lib.lib()
        _lib.check(L.nnconv_init())
        e = edge_index.size(1)
        ws_b, tmp_b = ctypes.c_size_t(), ctypes.c_size_t()
        _lib.check(L.nnconv_plan_sizes(e, n_nodes, ctypes.byref(ws_b), ctypes.byref(tmp_b)))
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
        _lib.check(L.nnconv_plan_create(_ptr(row0), _ptr(row1), e, n_nodes, _lib.FLOW[flow], _ptr(self.ws),
                                        ws_b.value, _ptr(tmp), tmp_b.value, _stream_ptr(dev), ctypes.byref(h)))
        self.handle = h
        self.key = _plan_key(edge_index, n_nodes, flow)
        self.nbytes = self.ws.numel() + edge_index.numel() * edge_index.element_size()
        info = (ctypes.c_int64 * 8)()
        _lib.check(L.nnconv_plan_info(h, info, 8))
        self.E, self.N, self.n_src, self.n_tiles, self.max_out_deg, self.src_sorted = [int(v) for v in info[:6]]
        stats['plans_built'] += 1
        self._finalizer = weakref.finalize(self, L.nnconv_plan_destroy, h)


class _Streamed(object):
    """Partially resident edge features: h of the sorted edges [0, E_res) (``h_res``, nnconv_edge_features_prefix);
    every application recomputes the other edges' h in ``n_chunks`` chunks from ``ea32`` (nnconv_apply_streamed)."""

    def __init__(self, h_res, E_res, ws_bytes, n_chunks, ea32):
        self.h_res, self.E_res, self.ws_bytes, self.n_chunks, self.ea32 = h_res, E_res, ws_bytes, n_chunks, ea32


def _streamed_chunks(plan, prepared, e_res, n_apps, ws_bytes):
    """Source batches whose edge features a streamed backward call recomputes (n_apps = 0: the per-application call)."""
    n = ctypes.c_int64(0)
    _lib.check(_lib.lib().nnconv_backward_streamed_chunks(plan.handle, prepared.handle, e_res, n_apps, ws_bytes,
                                                          ctypes.byref(n)))
    return n.value


def _plan_key(edge_index, n_nodes, flow):
    return (edge_index.data_ptr(), tuple(edge_index.shape), tuple(edge_index.stride()), edge_index._version,
            edge_index.device.index, int(n_nodes), flow)


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


def _linear_chain(nn_module):
    """The edge network must be the reference's DenseNet shape: Linear (ReLU Linear)* with no output
    nonlinearity (graph-neural-operator/utilities.py:201-227; every call site passes torch.nn.ReLU,
    normalize=False)."""
    mods = [m for m in nn_module.modules() if len(list(m.children())) == 0]
    lin = []
    expect_linear = True
    for m in mods:
        if isinstance(m, torch.nn.Linear):
            if not expect_linear:
                raise NotImplementedError('edge network: two Linear layers without a ReLU in between')
            if m.bias is None:
                raise NotImplementedError('edge network: Linear without bias is not supported')
            lin.append(m)
            expect_linear = False
        elif isinstance(m, torch.nn.ReLU):
            if expect_linear:
                raise NotImplementedError('edge network: ReLU must follow a Linear layer')
            expect_linear = True
        else:
            raise NotImplementedError('edge network: only Linear/ReLU chains (DenseNet) are supported, found %s'
                                      % type(m).__name__)
    if not lin or expect_linear:
        raise NotImplementedError('edge network must end with a Linear layer (no output nonlinearity)')
    return lin


class _Prepared(object):
    """nnconv_weights_t: padded / permuted / down-converted snapshot of the edge-MLP parameters."""

    def __init__(self, linears, cin, cout, precision):
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
        _lib.check(L.nnconv_weights_create(n, c_dims, cin, cout, prec, wp, bp, _ptr(self.buf), nbytes.value,
                                           _stream_ptr(dev), ctypes.byref(h)))
        self._keep = (ws, bs)
        self.handle = h
        self.dims = dims
        self.precision = precision
        self.tc = bool(L.nnconv_weights_tc_supported(h))
        self.bwd_tc = bool(L.nnconv_backward_tc_supported(h))
        stats['weight_preps'] += 1
        stats['launches'] += 2 * n + 1
        self._finalizer = weakref.finalize(self, L.nnconv_weights_destroy, h)


class _NNConvFunction(torch.autograd.Function):
    """Differentiable wrapper, CUDA-core variant: forward = the configured precision path, backward =
    nnconv_backward_ex (fp32 CUDA-core kernels, csrc/backward.cu; any shape, activations recomputed).  Gradients flow
    to x, edge_attr, the edge-MLP Linear weights/biases, root and bias; edge_index gets none."""

    @staticmethod
    def forward(ctx, module, x, edge_index, edge_attr, *params):
        ctx.module = module
        ctx.edge_index = edge_index
        ctx.save_for_backward(x, edge_attr)
        return module._forward_impl(x, edge_index, edge_attr, for_grad=True)

    @staticmethod
    def backward(ctx, grad_out):
        module = ctx.module
        x, edge_attr = ctx.saved_tensors
        grads = module._backward_impl(x, ctx.edge_index, edge_attr, grad_out, want_ea=ctx.needs_input_grad[3])
        # order of *params in forward(): list(module.parameters())
        by_id = {id(p): g for p, g in grads['params']}
        return (None, grads['x'] if ctx.needs_input_grad[1] else None, None, grads.get('edge_attr')) + tuple(
            by_id.get(id(p)) for p in module.parameters())


class _TrainState(object):
    """What the tensor-core backward shares between the applications of one conv on one (edge_attr, parameters):
    the plan, the prepared weights, the cached edge features and, filled during the backward sweep, every
    application's (grad_out, x) for the ONE deferred pass through the hidden layers."""

    def __init__(self, key, plan, prepared, h, ea32):
        self.key, self.plan, self.prepared, self.h, self.ea32 = key, plan, prepared, h, ea32
        self.apps = []
        self.consumed = False
        self.token = None
        self.acts = None            # hidden activations kept by the forward (nnconv_edge_features_keep), or None


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
        return torch.zeros(1, device=state.ea32.device)

    @staticmethod
    def backward(ctx, _):
        state = ctx.state
        grads, gea = ctx.module._backward_mlp_impl(state, want_ea=ctx.needs_input_grad[2])
        state.consumed = True
        state.apps = []
        state.h = state.ea32 = state.acts = None     # the per-edge buffers are no longer pinned by this (finished) graph
        return (None, None, gea.to(ctx.ea_dtype) if gea is not None else None) + tuple(grads)


class _ApplyFn(torch.autograd.Function):
    """One NNConv application given the edge features (tensor-core forward and backward)."""

    @staticmethod
    def forward(ctx, module, state, x, token, w_last, b_last, root, bias):
        ctx.module, ctx.state = module, state
        x32 = x.detach().contiguous().float()
        ctx.save_for_backward(x32)
        ctx.x_dtype = x.dtype
        return module._apply_impl(state.plan, state.prepared, state.h, x32)

    @staticmethod
    def backward(ctx, grad_out):
        (x32,) = ctx.saved_tensors
        module, state = ctx.module, ctx.state
        g32 = grad_out.detach().contiguous().float()
        dx, dwl, dbl, droot, dbias = module._backward_apply_impl(state, x32, g32)
        state.apps.append((g32, x32))
        return (None, None, dx.to(ctx.x_dtype) if ctx.needs_input_grad[2] else None, torch.zeros_like(state.token),
                dwl, dbl, droot, dbias)


class NNConv_old(torch.nn.Module):
    r"""Edge-conditioned convolution  x'_i = Theta x_i + aggr_{j in N(i)} x_j . h_Theta(e_ij)
    (reference docstring: graph-neural-operator/nn_conv.py:198-232).

    Args are the reference's (nn_conv.py:234-241).  Extra keyword ``precision`` in
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
        self._prepared = None
        self._prepared_key = None
        self._h_cache = collections.OrderedDict()
        self._h_cache_max = 1
        self._k_cache = None
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
        bound = 1.0 / math.sqrt(self.in_channels)
        if self.root is not None:
            self.root.data.uniform_(-bound, bound)
        if self.bias is not None:
            self.bias.data.uniform_(-bound, bound)

    # -- reference: nn_conv.py:267-271 ------------------------------------------------------------------
    def forward(self, x, edge_index, edge_attr):
        x = x.unsqueeze(-1) if x.dim() == 1 else x
        pseudo = edge_attr.unsqueeze(-1) if edge_attr.dim() == 1 else edge_attr
        needs_grad = torch.is_grad_enabled() and (
            x.requires_grad or pseudo.requires_grad or any(p.requires_grad for p in self.parameters()))
        if needs_grad:
            if self.aggr == 'max':
                raise NotImplementedError("aggr='max' is used by no call site of the reference and is not built")
            state = self._train_state(x, edge_index, pseudo)
            if state is not None:            # tensor-core backward (csrc/backward_tc.cu)
                lin = _linear_chain(self.nn)[-1]
                return _ApplyFn.apply(self, state, x, state.token, lin.weight, lin.bias, self.root, self.bias)
            return _NNConvFunction.apply(self, x, edge_index, pseudo, *list(self.parameters()))
        return self._forward_impl(x, edge_index, pseudo)

    def __repr__(self):
        return '{}({}, {})'.format(self.__class__.__name__, self.in_channels, self.out_channels)

    # -- cache control ----------------------------------------------------------------------------------
    def invalidate(self):
        """Drop the prepared-weight snapshots and cached edge features (needed after parameter writes that do
        not bump the tensors' version counters, e.g. through ``.data``)."""
        self._prepared = None
        self._prepared_key = None
        self._prepared32_key = None
        self._prepared32 = None
        self._h_cache.clear()
        self._k_cache = None

    def train(self, mode=True):
        self.invalidate()
        return super(NNConv_old, self).train(mode)

    def _load_from_state_dict(self, *args, **kwargs):
        self.invalidate()
        return super(NNConv_old, self)._load_from_state_dict(*args, **kwargs)

    # -- host-side sequencing ---------------------------------------------------------------------------
    def _get_prepared(self, precision):
        linears = _linear_chain(self.nn)
        key = (precision,) + tuple((l.weight.data_ptr(), l.weight._version, l.bias.data_ptr(), l.bias._version)
                                   for l in linears)
        if self._prepared is None or self._prepared_key != key:
            self._prepared = _Prepared(linears, self.in_channels, self.out_channels, precision)
            self._prepared_key = key
            self._h_cache.clear()
            self._k_cache = None
        return self._prepared

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
        """x-independent part of message(): cached across the T applications of a shared conv.  keep_acts (training):
        also keep the hidden activations for the backward (returned by ``kept_acts``).  Returns h, or a _Streamed
        when only a prefix of h fits (see the class docstring)."""
        key = (plan.key, edge_attr.data_ptr(), tuple(edge_attr.shape), edge_attr._version, id(prepared))
        hit = self._h_cache.get(key)
        L = _lib.lib()
        acts_b = ctypes.c_size_t(0)
        if keep_acts:
            _lib.check(L.nnconv_edge_acts_sizes(plan.handle, prepared.handle, ctypes.byref(acts_b)))
            if acts_b.value > _KEEP_ACTS_MAX_BYTES:
                acts_b = ctypes.c_size_t(0)
        streamed_hit = hit is not None and isinstance(hit[0], _Streamed)
        if streamed_hit and for_grad:
            if not self.streamed_training:
                self._streaming_grad_error(hit[0].h_res.numel())
            if hit[0].auto and not hit[0].for_grad:
                hit = None               # sized for inference: the prefix leaves no room for the backward's workspace
        if hit is not None and (acts_b.value == 0 or hit[2] is not None or streamed_hit):
            return hit[0]
        h_b, ws_b = ctypes.c_size_t(), ctypes.c_size_t()
        _lib.check(L.nnconv_edge_features_sizes(plan.handle, prepared.handle, _EF_WS_BYTES, ctypes.byref(h_b),
                                                ctypes.byref(ws_b)))
        dev = edge_attr.device
        self._h_cache.clear()                       # free the previous sample's features first
        self._k_cache = None
        budget = self._budget()
        streams = self._streams(plan, prepared)
        if budget is not None and h_b.value > budget and streams:
            if for_grad and not self.streamed_training:
                self._streaming_grad_error(budget)
            return self._streamed_features(key, plan, prepared, edge_attr, budget, for_grad)
        try:
            h = torch.empty(h_b.value, dtype=torch.uint8, device=dev)
            ws = torch.empty(ws_b.value, dtype=torch.uint8, device=dev)
        except torch.cuda.OutOfMemoryError:
            if not streams:
                raise
            h = ws = None
            if for_grad and not self.streamed_training:
                self._streaming_grad_error(h_b.value)
            self._h_cache.clear()
            self._k_cache = None
            self._tstate = None
            return self._streamed_features(key, plan, prepared, edge_attr, None, for_grad)
        acts = torch.empty(acts_b.value, dtype=torch.uint8, device=dev) if acts_b.value else None
        n_l = ctypes.c_int64(0)
        if acts is not None:
            _lib.check(L.nnconv_edge_features_keep(plan.handle, prepared.handle, _ptr(edge_attr), _ptr(h), _ptr(acts),
                                                   _ptr(ws), ws_b.value, _stream_ptr(dev), ctypes.byref(n_l)))
        else:
            _lib.check(L.nnconv_edge_features(plan.handle, prepared.handle, _ptr(edge_attr), _ptr(h), _ptr(ws),
                                              ws_b.value, _stream_ptr(dev), ctypes.byref(n_l)))
        stats['launches'] += n_l.value
        stats['edge_feature_passes'] += 1
        self._check_overflow(prepared, ws, dev)
        self._h_cache[key] = (h, edge_attr, acts)    # hold edge_attr so its address cannot be recycled
        return h

    @staticmethod
    def _streaming_grad_error(nbytes):
        raise RuntimeError(
            'graph_pde_b200.NNConv: the edge features of this graph do not fit on the device or in the cache budget '
            '(%d bytes), and training needs the whole h resident: streamed edge features are inference only (call '
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
            _lib.check(_lib.lib().nnconv_backward_sizes(plan.handle, self._get_prepared32().handle, _BWD_WS_BYTES,
                                                        ctypes.byref(b)))
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

    def _streamed_features(self, key, plan, prepared, edge_attr, budget, for_grad=False):
        """Cache the unit-aligned prefix of h that fits ``budget`` bytes (None: what the device has free beside the
        streaming workspace and, for training, the backward's workspace) and return the _Streamed the applications run
        from."""
        L = _lib.lib()
        dev = edge_attr.device

        def split(b):
            e_res, h_b, ws_b, n_ch = ctypes.c_int64(), ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_int64()
            _lib.check(L.nnconv_stream_split(plan.handle, prepared.handle, max(int(b), 0), _EF_WS_BYTES,
                                             ctypes.byref(e_res), ctypes.byref(h_b), ctypes.byref(ws_b),
                                             ctypes.byref(n_ch)))
            return e_res.value, h_b.value, ws_b.value, n_ch.value

        e_res, h_b, ws_b, n_ch = split(budget if budget is not None else 0)
        if budget is None:
            free = torch.cuda.mem_get_info(dev)[0] + torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)
            work = ws_b + _STREAM_MARGIN_BYTES
            if for_grad:
                # the streamed backward's workspaces do not depend on where the prefix ends: sized at E_res = 0
                work += self._backward_reserve(plan, prepared, 0, edge_attr) + _STREAM_TRAIN_MARGIN_BYTES
            e_res, h_b, ws_b, n_ch = split(free - work)
        # training on the tensor cores: the backward's workspace (several GiB: 9 GiB at 241^2, f16x2) is allocated here,
        # beside the prefix, and reused by every backward call of this step.  Allocated per call, it would need one
        # contiguous block of that size after the forward has fragmented the caching allocator's segments.
        bwd_ws = None
        if for_grad and _BWD_MODE != 'fp32' and prepared.bwd_tc:
            # sized at E_res = 0: the streamed sizes do not depend on where the prefix ends, and they bound the whole-h
            # sizes should the prefix below end up covering every edge
            bwd_ws = torch.empty(self._tc_backward_ws_bytes(plan, prepared, 0), dtype=torch.uint8, device=dev)
        h_res = None
        if e_res > 0:
            try:
                h_res = torch.empty(h_b, dtype=torch.uint8, device=dev)
            except torch.cuda.OutOfMemoryError:
                if budget is not None:
                    raise
                e_res, h_b, ws_b, n_ch = split(0)
        if h_res is None:
            h_res = torch.empty(0, dtype=torch.uint8, device=dev)
        if e_res > 0:
            ef_h, ef_ws = ctypes.c_size_t(), ctypes.c_size_t()
            _lib.check(L.nnconv_edge_features_sizes(plan.handle, prepared.handle, _EF_WS_BYTES, ctypes.byref(ef_h),
                                                    ctypes.byref(ef_ws)))
            ws = torch.empty(ef_ws.value, dtype=torch.uint8, device=dev)
            n_l = ctypes.c_int64(0)
            _lib.check(L.nnconv_edge_features_prefix(plan.handle, prepared.handle, _ptr(edge_attr), e_res, _ptr(h_res),
                                                     _ptr(ws), ef_ws.value, _stream_ptr(dev), ctypes.byref(n_l)))
            stats['launches'] += n_l.value
            stats['edge_feature_passes'] += 1
            self._check_overflow(prepared, ws, dev)
            del ws
        st = _Streamed(h_res, e_res, ws_b, n_ch, edge_attr)
        st.auto, st.for_grad, st.bwd_ws = budget is None, for_grad, bwd_ws
        self._h_cache[key] = (st, edge_attr, None)
        return st

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

    def kept_acts(self, h):
        for ent in self._h_cache.values():
            if ent[0] is h:
                return ent[2]
        return None

    def _check_inputs(self, x, edge_index, pseudo):
        _require_cuda(x, 'x')
        _require_cuda(edge_index, 'edge_index')
        _require_cuda(pseudo, 'edge_attr')
        if self.aggr == 'max':
            raise NotImplementedError("aggr='max' is used by no call site of the reference and is not built")
        if edge_index.dtype != torch.int64 or edge_index.dim() != 2 or edge_index.size(0) != 2:
            raise ValueError('edge_index must be an int64 tensor of shape [2, E]')
        if x.size(1) != self.in_channels:
            raise ValueError('x has %d channels, expected %d' % (x.size(1), self.in_channels))
        if pseudo.size(0) != edge_index.size(1):
            raise ValueError('edge_attr has %d rows for %d edges' % (pseudo.size(0), edge_index.size(1)))

    def _prepare(self, x, edge_index, pseudo, keep_acts=False, for_grad=False):
        """plan, prepared weights, fp32 edge_attr and the (cached) edge features for this call."""
        precision = self.precision or default_precision()
        ea32 = pseudo.detach()
        if ea32.dtype != torch.float32 or not ea32.is_contiguous():
            ea32 = ea32.contiguous().float()
        plan = get_plan(edge_index, x.size(0), self.flow)
        prepared = self._get_prepared(precision)
        h = self.edge_features(plan, prepared, ea32, keep_acts and prepared.bwd_tc, for_grad)
        return plan, prepared, ea32, h

    def _wants_edge_kernels(self, plan, prepared):
        """The graph-shape policy of formulation B (see _edge_kernels)."""
        if _EDGE_KERNELS == 'off' or prepared.precision not in ('f16', 'fp16', 'bf16') or plan.E == 0:
            return False
        return _EDGE_KERNELS == 'on' or ((plan.E <= _EDGE_KERNELS_MAX_DEG * max(plan.n_src, 1) or
                                          plan.E <= _EDGE_KERNELS_MAX_EDGES) and
                                         plan.E * self.in_channels * self.out_channels * 2 <= _EDGE_KERNELS_MAX_BYTES)

    def _edge_kernels(self, plan, prepared, h):
        """K_e = W_L h_e + b_L for every edge (formulation B) when the graph has few out-edges per source, else None.
        Cached with h: as x-independent as the edge features."""
        if isinstance(h, _Streamed) or not self._wants_edge_kernels(plan, prepared):
            return None
        hit = getattr(self, '_k_cache', None)
        if hit is not None and hit[0] is h:
            return hit[1]
        if _CAPTURE_SINK is not None and plan.key in self._kmat_overflowed:
            return None         # a captured step keeps the choice its eager warm-up made: formulation C
        L = _lib.lib()
        nbytes = ctypes.c_size_t()
        if L.nnconv_edge_kernels_sizes(plan.handle, prepared.handle, ctypes.byref(nbytes)) != _lib.OK:
            return None                                   # shape not covered: formulation C
        kmat = torch.empty(nbytes.value, dtype=torch.uint8, device=h.device)
        _lib.check(L.nnconv_edge_kernels(plan.handle, prepared.handle, _ptr(h), _ptr(kmat), _stream_ptr(h.device)))
        stats['launches'] += 1
        stats['edge_kernel_passes'] = stats.get('edge_kernel_passes', 0) + 1
        if self._overflow_count(prepared, kmat[nbytes.value - 1024:], h.device, edge_kernels=True):
            # K_e left the fp16 range (it holds b_L in 16 bits): formulation C, which keeps b_L in fp32 and whose h and
            # Y passed their own checks, computes these edges instead
            kmat = None
            self._kmat_overflowed.add(plan.key)
        self._k_cache = (h, kmat)
        return kmat

    def _apply_impl(self, plan, prepared, h, x32, flags=0):
        L = _lib.lib()
        dev = x32.device
        if isinstance(h, _Streamed):
            return self._apply_streamed(plan, prepared, h, x32, flags)
        kmat = self._edge_kernels(plan, prepared, h)
        if kmat is not None:
            out = torch.empty(x32.size(0), self.out_channels, dtype=torch.float32, device=dev)
            root = self.root.detach().contiguous().float() if self.root is not None else None
            bias = self.bias.detach().contiguous().float() if self.bias is not None else None
            _lib.check(L.nnconv_apply_edge_ex(plan.handle, prepared.handle, _ptr(kmat), _ptr(x32), _ptr(root), _ptr(bias),
                                              _lib.AGGR[self.aggr], flags, _ptr(out), _stream_ptr(dev)))
            stats['launches'] += 2
            stats['applies'] += 1
            return out
        ws_b = ctypes.c_size_t()
        _lib.check(L.nnconv_apply_sizes(plan.handle, prepared.handle, _Y_BYTES, ctypes.byref(ws_b)))
        ws = torch.empty(ws_b.value, dtype=torch.uint8, device=dev)
        out = torch.empty(x32.size(0), self.out_channels, dtype=torch.float32, device=dev)
        root = self.root.detach().contiguous().float() if self.root is not None else None
        bias = self.bias.detach().contiguous().float() if self.bias is not None else None
        n_l = ctypes.c_int64(0)
        _lib.check(L.nnconv_apply_ex(plan.handle, prepared.handle, _ptr(h), _ptr(x32), _ptr(root), _ptr(bias),
                                     _lib.AGGR[self.aggr], flags, _ptr(out), _ptr(ws), ws_b.value, _stream_ptr(dev),
                                     ctypes.byref(n_l)))
        stats['launches'] += n_l.value
        stats['applies'] += 1
        return out

    def _apply_streamed(self, plan, prepared, st, x32, flags):
        """One application with partially resident edge features (nnconv_apply_streamed): no allocation inside the
        library and, besides the optional overflow check, no host sync -- capturable by capture.GraphedForward."""
        L = _lib.lib()
        dev = x32.device
        ws = torch.empty(st.ws_bytes, dtype=torch.uint8, device=dev)
        out = torch.empty(x32.size(0), self.out_channels, dtype=torch.float32, device=dev)
        root = self.root.detach().contiguous().float() if self.root is not None else None
        bias = self.bias.detach().contiguous().float() if self.bias is not None else None
        n_l = ctypes.c_int64(0)
        _lib.check(L.nnconv_apply_streamed(plan.handle, prepared.handle, _ptr(st.ea32), _ptr(st.h_res), st.E_res,
                                           _ptr(x32), _ptr(root), _ptr(bias), _lib.AGGR[self.aggr], flags, _ptr(out),
                                           _ptr(ws), st.ws_bytes, _stream_ptr(dev), ctypes.byref(n_l)))
        stats['launches'] += n_l.value
        stats['applies'] += 1
        stats['streamed_chunk_passes'] += st.n_chunks
        if st.n_chunks:
            self._check_overflow(prepared, ws, dev)
        return out

    def _forward_impl(self, x, edge_index, pseudo, flags=0, for_grad=False):
        self._check_inputs(x, edge_index, pseudo)
        with torch.cuda.device(x.device):
            x32 = x.detach().contiguous().float()
            plan, prepared, _, h = self._prepare(x32, edge_index, pseudo, for_grad=for_grad)
            return self._apply_impl(plan, prepared, h, x32, flags)

    def residual_step(self, z, edge_index, edge_attr, relu_in=True):
        """One V-cycle step ``x <- relu(x + conv(x))`` (multipole-graph-neural-operator/neurips1_MGKN.py:76,81,84) on
        PRE-activations, inference only: with ``x = relu(z)`` (``x = z`` if not ``relu_in``) returns
        ``z' = x + conv(x)``; the caller chains ``z'`` into the next step and applies the last ReLU itself.  The ReLU
        and the residual live in the node-prep launch of the application (``nnconv_apply_ex``), so a chain of steps
        has no elementwise kernels between its applications."""
        if self.in_channels != self.out_channels:
            raise ValueError('residual_step needs in_channels == out_channels')
        if torch.is_grad_enabled() and (z.requires_grad or edge_attr.requires_grad or
                                        any(p.requires_grad for p in self.parameters())):
            raise RuntimeError('residual_step is a forward-only path: call it under torch.no_grad()')
        if self.aggr == 'max':
            raise NotImplementedError("aggr='max' is used by no call site of the reference and is not built")
        pseudo = edge_attr.unsqueeze(-1) if edge_attr.dim() == 1 else edge_attr
        flags = _lib.APPLY_RESIDUAL | (_lib.APPLY_RELU_IN if relu_in else 0)
        return self._forward_impl(z, edge_index, pseudo, flags)

    # -- tensor-core training path ----------------------------------------------------------------------
    def _train_state(self, x, edge_index, pseudo):
        """State shared by the applications of this conv on (edge_attr, parameters), or None when the tensor-core
        backward does not cover the configuration (the fp32 CUDA-core backward is used then)."""
        mode = _BWD_MODE
        if mode == 'fp32':
            return None
        self._check_inputs(x, edge_index, pseudo)
        with torch.cuda.device(x.device):
            plan, prepared, ea32, h = self._prepare(x, edge_index, pseudo, keep_acts=True, for_grad=True)
            if not prepared.bwd_tc:
                if mode == 'tc':
                    raise NotImplementedError('NNCONV_B200_BACKWARD=tc: shape / precision not covered by the tensor-core backward')
                return None
            # requires_grad is part of the key: a state whose token is not connected to edge_attr cannot serve an
            # application that must deliver its gradient
            key = (plan.key, ea32.data_ptr(), tuple(ea32.shape), ea32._version, id(prepared), pseudo.requires_grad)
            st = getattr(self, '_tstate', None)
            if st is None or st.key != key or st.consumed or st.h is not h:
                st = _TrainState(key, plan, prepared, h, ea32)
                st.acts = self.kept_acts(h)
                hidden = []
                for l in _linear_chain(self.nn)[:-1]:
                    hidden += [l.weight, l.bias]
                st.token = _EdgeFeaturesFn.apply(self, st, pseudo, *hidden)
                self._tstate = st
            return st

    def _backward_apply_impl(self, state, x32, g32):
        L = _lib.lib()
        dev = x32.device
        plan, prep = state.plan, state.prepared
        lin = _linear_chain(self.nn)[-1]
        with torch.cuda.device(dev):
            dx = torch.empty_like(x32)
            dwl = torch.empty_like(lin.weight, dtype=torch.float32)
            dbl = torch.empty_like(lin.bias, dtype=torch.float32)
            droot = torch.empty_like(self.root, dtype=torch.float32) if self.root is not None else None
            dbias = torch.empty_like(self.bias, dtype=torch.float32) if self.bias is not None else None
            root = self.root.detach().contiguous().float() if self.root is not None else None
            if isinstance(state.h, _Streamed):
                self._backward_apply_streamed(state, x32, g32, dx, dwl, dbl, root, droot, dbias)
            else:
                ws_b = ctypes.c_size_t()
                _lib.check(L.nnconv_backward_apply_sizes(plan.handle, prep.handle, _BWD_APPLY_WS_BYTES,
                                                         ctypes.byref(ws_b)))
                ws = torch.empty(ws_b.value, dtype=torch.uint8, device=dev)
                _lib.check(L.nnconv_backward_apply(plan.handle, prep.handle, _ptr(state.h), _ptr(x32), _ptr(root),
                                                   _lib.AGGR[self.aggr], _ptr(g32), _ptr(dx), _ptr(dwl), _ptr(dbl),
                                                   _ptr(droot), _ptr(dbias), _ptr(ws), ws_b.value, _stream_ptr(dev)))
            stats['backwards'] = stats.get('backwards', 0) + 1
        return dx, dwl, dbl, droot, dbias

    def _backward_apply_streamed(self, state, x32, g32, dx, dwl, dbl, root, droot, dbias):
        """nnconv_backward_apply over the resident prefix of h; the other edges' h is recomputed per source batch."""
        L = _lib.lib()
        dev = x32.device
        plan, prep, st = state.plan, state.prepared, state.h
        ws = self._streamed_bwd_ws(st, plan, prep, 0)
        n_l = ctypes.c_int64(0)
        _lib.check(L.nnconv_backward_apply_streamed(plan.handle, prep.handle, _ptr(st.ea32), _ptr(st.h_res), st.E_res,
                                                    _ptr(x32), _ptr(root), _lib.AGGR[self.aggr], _ptr(g32), _ptr(dx),
                                                    _ptr(dwl), _ptr(dbl), _ptr(droot), _ptr(dbias), _ptr(ws), ws.numel(),
                                                    _stream_ptr(dev), ctypes.byref(n_l)))
        stats['launches'] += n_l.value
        stats['streamed_backward_chunk_passes'] += _streamed_chunks(plan, prep, st.E_res, 0, ws.numel())

    @staticmethod
    def _streamed_bwd_ws(st, plan, prep, n_apps):
        """The workspace allocated with the prefix (see _streamed_features), else one of the size the call needs
        (n_apps = 0: a per-application call)."""
        if st.bwd_ws is not None:
            return st.bwd_ws
        L = _lib.lib()
        b = ctypes.c_size_t()
        if n_apps == 0:
            _lib.check(L.nnconv_backward_apply_streamed_sizes(plan.handle, prep.handle, st.E_res, _BWD_APPLY_WS_BYTES,
                                                              _EF_WS_BYTES, ctypes.byref(b)))
        else:
            _lib.check(L.nnconv_backward_mlp_streamed_sizes(plan.handle, prep.handle, st.E_res, n_apps,
                                                            _BWD_MLP_WS_BYTES, ctypes.byref(b)))
        return torch.empty(b.value, dtype=torch.uint8, device=st.h_res.device)

    def _backward_mlp_impl(self, state, want_ea=False):
        """Gradients of the hidden Linear layers, one pass for all applications recorded in the state (in groups
        of <= 6 when a conv is applied more often), and with ``want_ea`` the fp32 gradient w.r.t. edge_attr
        ([E, k_in], summed over the groups; else None)."""
        L = _lib.lib()
        plan, prep = state.plan, state.prepared
        hidden = _linear_chain(self.nn)[:-1]
        dev = state.ea32.device
        streamed = state.h if isinstance(state.h, _Streamed) else None
        total = None
        gea_total = None
        with torch.cuda.device(dev):
            for i0 in range(0, len(state.apps), _MLP_GROUP):
                apps = state.apps[i0:i0 + _MLP_GROUP]
                n = len(apps)
                if streamed is not None:
                    ws = self._streamed_bwd_ws(streamed, plan, prep, n)
                else:
                    ws_b = ctypes.c_size_t()
                    _lib.check(L.nnconv_backward_mlp_sizes(plan.handle, prep.handle, n, _BWD_MLP_WS_BYTES,
                                                           ctypes.byref(ws_b)))
                    ws = torch.empty(ws_b.value, dtype=torch.uint8, device=dev)
                dws = [torch.empty_like(l.weight, dtype=torch.float32) for l in hidden]
                dbs = [torch.empty_like(l.bias, dtype=torch.float32) for l in hidden]
                gea = torch.empty(state.ea32.shape, dtype=torch.float32, device=dev) if want_ea else None
                gp = (ctypes.c_void_p * n)(*[g.data_ptr() for g, _ in apps])
                xp = (ctypes.c_void_p * n)(*[x.data_ptr() for _, x in apps])
                wp = (ctypes.c_void_p * len(hidden))(*[t.data_ptr() for t in dws])
                bp = (ctypes.c_void_p * len(hidden))(*[t.data_ptr() for t in dbs])
                if streamed is not None:
                    _lib.check(L.nnconv_backward_mlp_streamed(plan.handle, prep.handle, _ptr(state.ea32),
                                                              _ptr(streamed.h_res), streamed.E_res, n, gp, xp,
                                                              _lib.AGGR[self.aggr], wp, bp, _ptr(ws), ws.numel(),
                                                              _stream_ptr(dev), _ptr(gea)))
                    stats['streamed_backward_chunk_passes'] += _streamed_chunks(plan, prep, streamed.E_res, n,
                                                                                ws.numel())
                else:
                    _lib.check(L.nnconv_backward_mlp_ex(plan.handle, prep.handle, _ptr(state.ea32), _ptr(state.h), n,
                                                        gp, xp, _lib.AGGR[self.aggr], wp, bp, _ptr(ws), ws_b.value,
                                                        _stream_ptr(dev), _ptr(getattr(state, 'acts', None)), _ptr(gea)))
                flat = [t for pair in zip(dws, dbs) for t in pair]
                total = flat if total is None else [a + b for a, b in zip(total, flat)]
                if gea is not None:
                    gea_total = gea if gea_total is None else gea_total + gea
            stats['mlp_backwards'] = stats.get('mlp_backwards', 0) + 1
        if total is None:     # no application contributed (cannot happen through autograd, kept for safety)
            total = [torch.zeros_like(p, dtype=torch.float32) for l in hidden for p in (l.weight, l.bias)]
            if want_ea:
                gea_total = torch.zeros(state.ea32.shape, dtype=torch.float32, device=dev)
        return total, gea_total

    def _get_prepared32(self):
        """fp32 weight snapshot of the CUDA-core backward (cached per parameter versions)."""
        linears = _linear_chain(self.nn)
        key = ('fp32',) + tuple((l.weight.data_ptr(), l.weight._version, l.bias.data_ptr(), l.bias._version)
                                for l in linears)
        if getattr(self, '_prepared32_key', None) != key:
            self._prepared32 = _Prepared(linears, self.in_channels, self.out_channels, 'fp32')
            self._prepared32_key = key
        return self._prepared32

    def _backward_impl(self, x, edge_index, pseudo, grad_out, want_ea=False):
        """fp32 CUDA-core backward of one application; with ``want_ea`` also the gradient w.r.t. edge_attr
        (returned under 'edge_attr' in pseudo's dtype)."""
        L = _lib.lib()
        with torch.cuda.device(x.device):
            x32 = x.detach().contiguous().float()
            ea32 = pseudo.detach().contiguous().float()
            g32 = grad_out.detach().contiguous().float()
            n = x32.size(0)
            plan = get_plan(edge_index, n, self.flow)
            linears = _linear_chain(self.nn)
            prep = self._get_prepared32()
            ws_b = ctypes.c_size_t()
            _lib.check(L.nnconv_backward_sizes(plan.handle, prep.handle, _BWD_WS_BYTES, ctypes.byref(ws_b)))
            ws = torch.empty(ws_b.value, dtype=torch.uint8, device=x.device)
            dx = torch.empty_like(x32)
            dws = [torch.empty_like(l.weight, dtype=torch.float32) for l in linears]
            dbs = [torch.empty_like(l.bias, dtype=torch.float32) for l in linears]
            droot = torch.empty_like(self.root, dtype=torch.float32) if self.root is not None else None
            dbias = torch.empty_like(self.bias, dtype=torch.float32) if self.bias is not None else None
            nl = len(linears)
            wp = (ctypes.c_void_p * nl)(*[t.data_ptr() for t in dws])
            bp = (ctypes.c_void_p * nl)(*[t.data_ptr() for t in dbs])
            root = self.root.detach().contiguous().float() if self.root is not None else None
            gea = torch.empty_like(ea32) if want_ea else None
            _lib.check(L.nnconv_backward_ex(plan.handle, prep.handle, _ptr(ea32), _ptr(x32), _ptr(root),
                                            _lib.AGGR[self.aggr], _ptr(g32), _ptr(dx), wp, bp, _ptr(droot), _ptr(dbias),
                                            _ptr(ws), ws_b.value, _stream_ptr(x.device), _ptr(gea)))
            stats['backwards'] = stats.get('backwards', 0) + 1
        params = [(l.weight, dw) for l, dw in zip(linears, dws)] + [(l.bias, db) for l, db in zip(linears, dbs)]
        if self.root is not None:
            params.append((self.root, droot))
        if self.bias is not None:
            params.append((self.bias, dbias))
        grads = {'x': dx.to(x.dtype), 'params': params}
        if gea is not None:
            grads['edge_attr'] = gea.to(pseudo.dtype)
        return grads


class NNConv(NNConv_old):
    """Drop-in for upstream ``torch_geometric.nn.NNConv`` as the MGKN scripts use it
    (multipole-graph-neural-operator/neurips1_MGKN.py:41,49,57; MGKN_general_darcy2d.py:45,53,61;
    MGKN_orthogonal_burgers1d.py:37).  NOTE: graph-neural-operator/nn_conv.py:8-96 also defines a class
    called NNConv (diagonal-kernel variant) which no script instantiates; it is out of scope."""
    pass


ECConv = NNConv
