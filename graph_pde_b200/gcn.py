"""GCNConv: the graph convolution of the reference's GCN baseline (multipole-graph-neural-operator/neurips4_GCN.py,
``from torch_geometric.nn import GCNConv``), with the PyG 1.x signature, parameters and normalisation:

    out = D^-1/2 (A + fill I) D^-1/2 x W + bias

Self loops follow PyG's ``add_remaining_self_loops``: a caller's self loops leave the edge list and every node gets
exactly one loop, of weight 1 if the caller's list had one, else ``fill`` (2 when ``improved``, else 1).  Degrees are
summed at the target; ``deg^-1/2`` is 0 for a zero degree; duplicate edges count once each.  ``normalize=False``: the
plain sum over the caller's edges (its loops included), no loops added; ``add_self_loops=False``: normalised without
added loops.  The library computes ``(A_hat x) W`` -- aggregation first, the same map re-associated -- in one
tensor-core kernel per application (csrc/gcn.cu, DESIGN 4.8); precision 'fp32' and shapes outside in, out in
{16, 32, ..., 128} run on the CUDA cores.  Forward and backward are bitwise reproducible run to run.

``cached=True`` is accepted: the graph (CSRs and norms) is cached per ``edge_index`` anyway, like the NNConv plans, so
PyG's behaviour of reusing the first graph forever is not reproduced.  ``edge_weight`` is not supported.
"""
import collections
import ctypes
import math
import weakref

import torch
from torch.nn import Parameter

from . import _lib
from . import nn_conv as _nc

__all__ = ['GCNConv', 'get_gcn_graph', 'stats']

# GCNConv's own counters; its kernel launches also count in nn_conv.stats['launches'] (every launch of the library)
stats = {'graphs_built': 0, 'applies': 0, 'backwards': 0}

# bounded like the NNConv plan cache, by entries and by bytes (graph buffers + the pinned edge_index); emptied by
# nn_conv.clear_caches()
_GRAPH_CACHE = collections.OrderedDict()
_GRAPH_CACHE_MAX = _nc._PLAN_CACHE_MAX
_GRAPH_CACHE_MAX_BYTES = _nc._PLAN_CACHE_MAX_BYTES


class _GcnGraph(object):
    """The library's graph of one (edge_index, n_nodes, flow, flags) and the buffer it lives in."""

    def __init__(self, edge_index, n_nodes, flow, flags):
        L = _lib.lib()
        _lib.check(L.nnconv_init())
        e = edge_index.size(1)
        ws_b, tmp_b = ctypes.c_size_t(), ctypes.c_size_t()
        _lib.check(L.nnconv_gcn_graph_sizes(e, n_nodes, ctypes.byref(ws_b), ctypes.byref(tmp_b)))
        dev = edge_index.device
        self.ws = torch.empty(ws_b.value, dtype=torch.uint8, device=dev)
        tmp = torch.empty(tmp_b.value, dtype=torch.uint8, device=dev)
        row0, row1 = edge_index[0].contiguous(), edge_index[1].contiguous()
        self.edge_index = edge_index          # keeps the storage (and so the cache key) alive
        h = ctypes.c_void_p()
        _lib.check(L.nnconv_gcn_graph_create(_nc._ptr(row0), _nc._ptr(row1), e, n_nodes, _lib.FLOW[flow], flags,
                                             _nc._ptr(self.ws), ws_b.value, _nc._ptr(tmp), tmp_b.value,
                                             _nc._stream_ptr(dev), ctypes.byref(h)))
        self.handle = h
        self.N = int(n_nodes)
        self.nbytes = self.ws.numel() + edge_index.numel() * edge_index.element_size()
        stats['graphs_built'] += 1
        self._finalizer = weakref.finalize(self, L.nnconv_gcn_graph_destroy, h)


def get_gcn_graph(edge_index, n_nodes, flow='source_to_target', flags=0):
    """The cached graph of ``edge_index`` (LRU keyed like the NNConv plans, plus the normalisation flags)."""
    key = _nc._plan_key(edge_index, n_nodes, flow) + (int(flags),)
    g = _GRAPH_CACHE.get(key)
    if g is None:
        g = _GcnGraph(edge_index, n_nodes, flow, flags)
        _GRAPH_CACHE[key] = g
        # the newest graph always stays
        while len(_GRAPH_CACHE) > 1 and (len(_GRAPH_CACHE) > _GRAPH_CACHE_MAX or
                                         sum(v.nbytes for v in _GRAPH_CACHE.values()) > _GRAPH_CACHE_MAX_BYTES):
            _GRAPH_CACHE.popitem(last=False)
    else:
        _GRAPH_CACHE.move_to_end(key)
    if _nc._CAPTURE_SINK is not None:         # a captured graph reads these buffers for as long as it lives
        _nc._CAPTURE_SINK.plans[('gcn',) + key] = g
    return g


def _operand(t):
    """fp32, contiguous and 16-byte aligned (the kernels load rows 16 bytes at a time)."""
    t = _nc._f32(t)
    return t.clone() if t.data_ptr() % 16 else t


class _GCNFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, graph, prec, cin, cout):
        L = _lib.lib()
        x32, w32, b32 = _operand(x), _nc._f32(weight), _nc._f32(bias)
        dev = x32.device
        ws_b = ctypes.c_size_t()
        _lib.check(L.nnconv_gcn_apply_sizes(graph.handle, prec, cin, cout, ctypes.byref(ws_b)))
        ws = torch.empty(max(ws_b.value, 1), dtype=torch.uint8, device=dev)
        out = torch.empty(graph.N, cout, dtype=torch.float32, device=dev)
        n_l = ctypes.c_int64(0)
        _lib.check(L.nnconv_gcn_apply(graph.handle, prec, cin, cout, _nc._ptr(x32), _nc._ptr(w32), _nc._ptr(b32),
                                      _nc._ptr(out), _nc._ptr(ws), ws_b.value, _nc._stream_ptr(dev), ctypes.byref(n_l)))
        _nc.stats['launches'] += n_l.value
        stats['applies'] += 1
        ctx.save_for_backward(x32, w32)
        ctx.graph, ctx.prec, ctx.cin, ctx.cout, ctx.has_bias = graph, prec, cin, cout, bias is not None
        return out

    @staticmethod
    def backward(ctx, grad_out):
        L = _lib.lib()
        x32, w32 = ctx.saved_tensors
        g = _operand(grad_out)
        dev = g.device
        ws_b = ctypes.c_size_t()
        _lib.check(L.nnconv_gcn_backward_sizes(ctx.graph.handle, ctx.prec, ctx.cin, ctx.cout, ctypes.byref(ws_b)))
        ws = torch.empty(ws_b.value, dtype=torch.uint8, device=dev)
        dx = torch.empty(ctx.graph.N, ctx.cin, dtype=torch.float32, device=dev)
        dw = torch.empty(ctx.cin, ctx.cout, dtype=torch.float32, device=dev)
        db = torch.empty(ctx.cout, dtype=torch.float32, device=dev) if ctx.has_bias else None
        n_l = ctypes.c_int64(0)
        _lib.check(L.nnconv_gcn_backward(ctx.graph.handle, ctx.prec, ctx.cin, ctx.cout, _nc._ptr(x32), _nc._ptr(w32),
                                         _nc._ptr(g), _nc._ptr(dx), _nc._ptr(dw), _nc._ptr(db), _nc._ptr(ws),
                                         ws_b.value, _nc._stream_ptr(dev), ctypes.byref(n_l)))
        _nc.stats['launches'] += n_l.value
        stats['backwards'] += 1
        return dx, dw, db, None, None, None, None


class GCNConv(torch.nn.Module):
    r"""PyG 1.x ``GCNConv(in_channels, out_channels, improved=False, cached=False, add_self_loops=True,
    normalize=True, bias=True, **kwargs)``; extra keywords ``precision`` ('f16' default, 'bf16', 'f16x2', 'fp32'; see
    NNConv_old) and ``flow``.  Parameters ``weight [in, out]`` (glorot) and ``bias [out]`` (zeros).  A PyG 2.x state
    dict (``lin.weight [out, in]``) loads too.  ``forward(x, edge_index, edge_weight=None)``: ``edge_weight`` raises
    NotImplementedError.  16-bit precisions need in and out multiples of 16 in [16, 128]; other shapes raise
    NNConvLibraryError pointing at 'fp32'."""

    def __init__(self, in_channels, out_channels, improved=False, cached=False, add_self_loops=True, normalize=True,
                 bias=True, **kwargs):
        super(GCNConv, self).__init__()
        self.precision = kwargs.pop('precision', None)
        self.flow = kwargs.pop('flow', 'source_to_target')
        if kwargs:
            raise TypeError('unexpected keyword arguments %s' % sorted(kwargs))
        if self.flow not in _lib.FLOW:
            raise ValueError('flow must be source_to_target or target_to_source')
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.improved = improved
        self.cached = cached
        self.add_self_loops = add_self_loops
        self.normalize = normalize
        self.weight = Parameter(torch.Tensor(in_channels, out_channels))
        if bias:
            self.bias = Parameter(torch.Tensor(out_channels))
        else:
            self.register_parameter('bias', None)
        self.reset_parameters()

    def reset_parameters(self):
        stdv = math.sqrt(6.0 / (self.weight.size(-2) + self.weight.size(-1)))   # torch_geometric.nn.inits.glorot
        self.weight.data.uniform_(-stdv, stdv)
        if self.bias is not None:
            self.bias.data.fill_(0)

    @property
    def flags(self):
        f = _lib.GCN_IMPROVED if self.improved else 0
        if not self.add_self_loops:
            f |= _lib.GCN_NO_SELF_LOOPS
        if not self.normalize:
            f |= _lib.GCN_NO_NORMALIZE
        return f

    def forward(self, x, edge_index, edge_weight=None):
        if edge_weight is not None:
            raise NotImplementedError('GCNConv: edge_weight is not supported (every edge has weight 1)')
        _nc._require_cuda(x, 'x')
        _nc._require_cuda(edge_index, 'edge_index')
        if edge_index.dtype != torch.int64 or edge_index.dim() != 2 or edge_index.size(0) != 2:
            raise ValueError('edge_index must be an int64 tensor of shape [2, E]')
        if edge_index.device != x.device:
            raise ValueError('edge_index is on %s, x on %s' % (edge_index.device, x.device))
        if x.dim() != 2 or x.size(1) != self.in_channels:
            raise ValueError('GCNConv: x must be [N, %d], got %s' % (self.in_channels, tuple(x.shape)))
        prec = _lib.PREC[self.precision or _nc.default_precision()]
        graph = get_gcn_graph(edge_index, x.size(0), self.flow, self.flags)
        return _GCNFn.apply(x, self.weight, self.bias, graph, prec, self.in_channels, self.out_channels)

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        lin = prefix + 'lin.weight'            # PyG 2.x keeps W as a Linear: [out, in]
        if lin in state_dict and prefix + 'weight' not in state_dict:
            state_dict[prefix + 'weight'] = state_dict.pop(lin).t()
        return super(GCNConv, self)._load_from_state_dict(state_dict, prefix, *args, **kwargs)

    def __repr__(self):
        return '{}({}, {})'.format(self.__class__.__name__, self.in_channels, self.out_channels)
