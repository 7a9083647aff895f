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
import ctypes
import math
import os
import weakref

import torch
from torch.nn import Parameter

from . import _lib

__all__ = ['NNConv_old', 'NNConv', 'ECConv', 'stats', 'clear_caches', 'default_precision']

stats = {'launches': 0, 'plans_built': 0, 'edge_feature_passes': 0, 'applies': 0, 'weight_preps': 0}

_PLAN_CACHE = collections.OrderedDict()
_PLAN_CACHE_MAX = int(os.environ.get('NNCONV_B200_PLAN_CACHE', '64'))                 # entries
_PLAN_CACHE_MAX_BYTES = int(os.environ.get('NNCONV_B200_PLAN_CACHE_BYTES', str(2 << 30)))   # plan buffers + pinned edge_index
_OVERFLOW_CHECK = os.environ.get('NNCONV_B200_OVERFLOW_CHECK', '1') != '0'
_Y_BYTES = int(os.environ.get('NNCONV_B200_Y_BYTES', str(48 << 20)))       # Y ring: 3 x 128 sources at out=64, Kp=1024
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


def default_precision():
    return os.environ.get('NNCONV_B200_PRECISION', 'f16')


def clear_caches():
    _PLAN_CACHE.clear()


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


def _plan_key(edge_index, n_nodes, flow):
    return (edge_index.data_ptr(), tuple(edge_index.shape), tuple(edge_index.stride()), edge_index._version,
            edge_index.device.index, int(n_nodes), flow)


def get_plan(edge_index, n_nodes, flow='source_to_target'):
    key = _plan_key(edge_index, n_nodes, flow)
    plan = _PLAN_CACHE.get(key)
    if plan is not None:
        _PLAN_CACHE.move_to_end(key)
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
    nnconv_backward (fp32 CUDA-core kernels, csrc/backward.cu; any shape, activations recomputed).  Gradients flow
    to x, the edge-MLP Linear weights/biases, root and bias; edge_index / edge_attr are leaf inputs in every
    reference script and get none."""

    @staticmethod
    def forward(ctx, module, x, edge_index, edge_attr, *params):
        ctx.module = module
        ctx.edge_index = edge_index
        ctx.save_for_backward(x, edge_attr)
        return module._forward_impl(x, edge_index, edge_attr)

    @staticmethod
    def backward(ctx, grad_out):
        module = ctx.module
        x, edge_attr = ctx.saved_tensors
        grads = module._backward_impl(x, ctx.edge_index, edge_attr, grad_out)
        # order of *params in forward(): list(module.parameters())
        by_id = {id(p): g for p, g in grads['params']}
        return (None, grads['x'] if ctx.needs_input_grad[1] else None, None, None) + tuple(
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
    (grad_out, x) pair collected in the state, the hidden layers are differentiated once for all T applications."""

    @staticmethod
    def forward(ctx, module, state, *hidden_params):
        ctx.module, ctx.state = module, state
        return torch.zeros(1, device=state.h.device)

    @staticmethod
    def backward(ctx, _):
        state = ctx.state
        grads = ctx.module._backward_mlp_impl(state)
        state.consumed = True
        state.apps = []
        state.h = state.ea32 = state.acts = None     # the per-edge buffers are no longer pinned by this (finished) graph
        return (None, None) + tuple(grads)


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

    Caches: the down-converted weights and the x-independent edge features are cached per (parameter versions,
    edge_attr version).  Optimizer steps, ``load_state_dict`` and ``train()/eval()`` invalidate them; writes that
    bypass autograd's version counter (``p.data.copy_()``, ``p.data.clamp_()``) do NOT -- call ``invalidate()``
    after such writes.
    """

    def __init__(self, in_channels, out_channels, nn, aggr='add', root_weight=True, bias=True, **kwargs):
        super(NNConv_old, self).__init__()
        self.precision = kwargs.pop('precision', None)
        self.flow = kwargs.pop('flow', 'source_to_target')
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
            x.requires_grad or any(p.requires_grad for p in self.parameters()))
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

    def edge_features(self, plan, prepared, edge_attr, keep_acts=False):
        """x-independent part of message(): cached across the T applications of a shared conv.  keep_acts (training):
        also keep the hidden activations for the backward (returned by ``kept_acts``)."""
        key = (plan.key, edge_attr.data_ptr(), tuple(edge_attr.shape), edge_attr._version, id(prepared))
        hit = self._h_cache.get(key)
        L = _lib.lib()
        acts_b = ctypes.c_size_t(0)
        if keep_acts:
            _lib.check(L.nnconv_edge_acts_sizes(plan.handle, prepared.handle, ctypes.byref(acts_b)))
            if acts_b.value > _KEEP_ACTS_MAX_BYTES:
                acts_b = ctypes.c_size_t(0)
        if hit is not None and (acts_b.value == 0 or hit[2] is not None):
            return hit[0]
        h_b, ws_b = ctypes.c_size_t(), ctypes.c_size_t()
        _lib.check(L.nnconv_edge_features_sizes(plan.handle, prepared.handle, _EF_WS_BYTES, ctypes.byref(h_b),
                                                ctypes.byref(ws_b)))
        dev = edge_attr.device
        self._h_cache.clear()                       # free the previous sample's features first
        self._k_cache = None
        h = torch.empty(h_b.value, dtype=torch.uint8, device=dev)
        ws = torch.empty(ws_b.value, dtype=torch.uint8, device=dev)
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
        if _OVERFLOW_CHECK and prepared.precision in ('f16', 'fp16', 'f16x2') and \
                not torch.cuda.is_current_stream_capturing():
            cnt = ctypes.c_int64(0)
            _lib.check(L.nnconv_edge_features_overflow(_ptr(ws), _stream_ptr(dev), ctypes.byref(cnt)))
            if cnt.value:
                raise FloatingPointError(
                    'graph_pde_b200.NNConv: %d blocks of edge-MLP activations left the fp16 range (|h| > 65504 or '
                    "NaN); use precision='bf16' or 'fp32' for this parameter scale (NNCONV_B200_OVERFLOW_CHECK=0 "
                    'disables this check and its one host sync per edge-feature pass)' % cnt.value)
        self._h_cache[key] = (h, edge_attr, acts)    # hold edge_attr so its address cannot be recycled
        return h

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

    def _prepare(self, x, edge_index, pseudo, keep_acts=False):
        """plan, prepared weights, fp32 edge_attr and the (cached) edge features for this call."""
        precision = self.precision or default_precision()
        ea32 = pseudo.detach()
        if ea32.dtype != torch.float32 or not ea32.is_contiguous():
            ea32 = ea32.contiguous().float()
        plan = get_plan(edge_index, x.size(0), self.flow)
        prepared = self._get_prepared(precision)
        h = self.edge_features(plan, prepared, ea32, keep_acts and prepared.bwd_tc)
        return plan, prepared, ea32, h

    def _edge_kernels(self, plan, prepared, h):
        """K_e = W_L h_e + b_L for every edge (formulation B) when the graph has few out-edges per source, else None.
        Cached with h: as x-independent as the edge features."""
        if _EDGE_KERNELS == 'off' or prepared.precision not in ('f16', 'fp16', 'bf16') or plan.E == 0:
            return None
        if _EDGE_KERNELS != 'on' and not ((plan.E <= _EDGE_KERNELS_MAX_DEG * max(plan.n_src, 1) or
                                           plan.E <= _EDGE_KERNELS_MAX_EDGES) and
                                          plan.E * self.in_channels * self.out_channels * 2 <= _EDGE_KERNELS_MAX_BYTES):
            return None
        hit = getattr(self, '_k_cache', None)
        if hit is not None and hit[0] is h:
            return hit[1]
        L = _lib.lib()
        nbytes = ctypes.c_size_t()
        if L.nnconv_edge_kernels_sizes(plan.handle, prepared.handle, ctypes.byref(nbytes)) != _lib.OK:
            return None                                   # shape not covered: formulation C
        kmat = torch.empty(nbytes.value, dtype=torch.uint8, device=h.device)
        _lib.check(L.nnconv_edge_kernels(plan.handle, prepared.handle, _ptr(h), _ptr(kmat), _stream_ptr(h.device)))
        stats['launches'] += 1
        stats['edge_kernel_passes'] = stats.get('edge_kernel_passes', 0) + 1
        self._k_cache = (h, kmat)
        return kmat

    def _apply_impl(self, plan, prepared, h, x32, flags=0):
        L = _lib.lib()
        dev = x32.device
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

    def _forward_impl(self, x, edge_index, pseudo, flags=0):
        self._check_inputs(x, edge_index, pseudo)
        with torch.cuda.device(x.device):
            x32 = x.detach().contiguous().float()
            plan, prepared, _, h = self._prepare(x32, edge_index, pseudo)
            return self._apply_impl(plan, prepared, h, x32, flags)

    def residual_step(self, z, edge_index, edge_attr, relu_in=True):
        """One V-cycle step ``x <- relu(x + conv(x))`` (multipole-graph-neural-operator/neurips1_MGKN.py:76,81,84) on
        PRE-activations, inference only: with ``x = relu(z)`` (``x = z`` if not ``relu_in``) returns
        ``z' = x + conv(x)``; the caller chains ``z'`` into the next step and applies the last ReLU itself.  The ReLU
        and the residual live in the node-prep launch of the application (``nnconv_apply_ex``), so a chain of steps
        has no elementwise kernels between its applications."""
        if self.in_channels != self.out_channels:
            raise ValueError('residual_step needs in_channels == out_channels')
        if torch.is_grad_enabled() and (z.requires_grad or any(p.requires_grad for p in self.parameters())):
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
        if mode == 'fp32' or pseudo.requires_grad:
            return None
        self._check_inputs(x, edge_index, pseudo)
        with torch.cuda.device(x.device):
            plan, prepared, ea32, h = self._prepare(x, edge_index, pseudo, keep_acts=True)
            if not prepared.bwd_tc:
                if mode == 'tc':
                    raise NotImplementedError('NNCONV_B200_BACKWARD=tc: shape / precision not covered by the tensor-core backward')
                return None
            key = (plan.key, ea32.data_ptr(), tuple(ea32.shape), ea32._version, id(prepared))
            st = getattr(self, '_tstate', None)
            if st is None or st.key != key or st.consumed or st.h is not h:
                st = _TrainState(key, plan, prepared, h, ea32)
                st.acts = self.kept_acts(h)
                hidden = []
                for l in _linear_chain(self.nn)[:-1]:
                    hidden += [l.weight, l.bias]
                st.token = _EdgeFeaturesFn.apply(self, st, *hidden)
                self._tstate = st
            return st

    def _backward_apply_impl(self, state, x32, g32):
        L = _lib.lib()
        dev = x32.device
        plan, prep = state.plan, state.prepared
        lin = _linear_chain(self.nn)[-1]
        with torch.cuda.device(dev):
            ws_b = ctypes.c_size_t()
            _lib.check(L.nnconv_backward_apply_sizes(plan.handle, prep.handle, _BWD_APPLY_WS_BYTES, ctypes.byref(ws_b)))
            ws = torch.empty(ws_b.value, dtype=torch.uint8, device=dev)
            dx = torch.empty_like(x32)
            dwl = torch.empty_like(lin.weight, dtype=torch.float32)
            dbl = torch.empty_like(lin.bias, dtype=torch.float32)
            droot = torch.empty_like(self.root, dtype=torch.float32) if self.root is not None else None
            dbias = torch.empty_like(self.bias, dtype=torch.float32) if self.bias is not None else None
            root = self.root.detach().contiguous().float() if self.root is not None else None
            _lib.check(L.nnconv_backward_apply(plan.handle, prep.handle, _ptr(state.h), _ptr(x32), _ptr(root),
                                               _lib.AGGR[self.aggr], _ptr(g32), _ptr(dx), _ptr(dwl), _ptr(dbl),
                                               _ptr(droot), _ptr(dbias), _ptr(ws), ws_b.value, _stream_ptr(dev)))
            stats['backwards'] = stats.get('backwards', 0) + 1
        return dx, dwl, dbl, droot, dbias

    def _backward_mlp_impl(self, state):
        """Gradients of the hidden Linear layers, one pass for all applications recorded in the state (in groups
        of <= 6 when a conv is applied more often)."""
        L = _lib.lib()
        plan, prep = state.plan, state.prepared
        hidden = _linear_chain(self.nn)[:-1]
        dev = state.h.device
        total = None
        with torch.cuda.device(dev):
            for i0 in range(0, len(state.apps), 6):
                apps = state.apps[i0:i0 + 6]
                n = len(apps)
                ws_b = ctypes.c_size_t()
                _lib.check(L.nnconv_backward_mlp_sizes(plan.handle, prep.handle, n, _BWD_MLP_WS_BYTES, ctypes.byref(ws_b)))
                ws = torch.empty(ws_b.value, dtype=torch.uint8, device=dev)
                dws = [torch.empty_like(l.weight, dtype=torch.float32) for l in hidden]
                dbs = [torch.empty_like(l.bias, dtype=torch.float32) for l in hidden]
                gp = (ctypes.c_void_p * n)(*[g.data_ptr() for g, _ in apps])
                xp = (ctypes.c_void_p * n)(*[x.data_ptr() for _, x in apps])
                wp = (ctypes.c_void_p * len(hidden))(*[t.data_ptr() for t in dws])
                bp = (ctypes.c_void_p * len(hidden))(*[t.data_ptr() for t in dbs])
                _lib.check(L.nnconv_backward_mlp(plan.handle, prep.handle, _ptr(state.ea32), _ptr(state.h), n, gp, xp,
                                                 _lib.AGGR[self.aggr], wp, bp, _ptr(ws), ws_b.value, _stream_ptr(dev),
                                                 _ptr(getattr(state, 'acts', None))))
                flat = [t for pair in zip(dws, dbs) for t in pair]
                total = flat if total is None else [a + b for a, b in zip(total, flat)]
            stats['mlp_backwards'] = stats.get('mlp_backwards', 0) + 1
        if total is None:     # no application contributed (cannot happen through autograd, kept for safety)
            total = [torch.zeros_like(p, dtype=torch.float32) for l in hidden for p in (l.weight, l.bias)]
        return total

    def _backward_impl(self, x, edge_index, pseudo, grad_out):
        if pseudo.requires_grad:
            raise NotImplementedError('gradients w.r.t. edge_attr are not built (leaf input in the reference)')
        L = _lib.lib()
        with torch.cuda.device(x.device):
            x32 = x.detach().contiguous().float()
            ea32 = pseudo.detach().contiguous().float()
            g32 = grad_out.detach().contiguous().float()
            n = x32.size(0)
            plan = get_plan(edge_index, n, self.flow)
            linears = _linear_chain(self.nn)
            key = ('fp32',) + tuple((l.weight.data_ptr(), l.weight._version, l.bias.data_ptr(), l.bias._version)
                                    for l in linears)
            if getattr(self, '_prepared32_key', None) != key:
                self._prepared32 = _Prepared(linears, self.in_channels, self.out_channels, 'fp32')
                self._prepared32_key = key
            prep = self._prepared32
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
            _lib.check(L.nnconv_backward(plan.handle, prep.handle, _ptr(ea32), _ptr(x32), _ptr(root),
                                         _lib.AGGR[self.aggr], _ptr(g32), _ptr(dx), wp, bp, _ptr(droot), _ptr(dbias),
                                         _ptr(ws), ws_b.value, _stream_ptr(x.device)))
            stats['backwards'] = stats.get('backwards', 0) + 1
        params = [(l.weight, dw) for l, dw in zip(linears, dws)] + [(l.bias, db) for l, db in zip(linears, dbs)]
        if self.root is not None:
            params.append((self.root, droot))
        if self.bias is not None:
            params.append((self.bias, dbias))
        return {'x': dx.to(x.dtype), 'params': params}


class NNConv(NNConv_old):
    """Drop-in for upstream ``torch_geometric.nn.NNConv`` as the MGKN scripts use it
    (multipole-graph-neural-operator/neurips1_MGKN.py:41,49,57; MGKN_general_darcy2d.py:45,53,61;
    MGKN_orthogonal_burgers1d.py:37).  NOTE: graph-neural-operator/nn_conv.py:8-96 also defines a class
    called NNConv (diagonal-kernel variant) which no script instantiates; it is out of scope."""
    pass


ECConv = NNConv
