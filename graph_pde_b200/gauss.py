"""The Gaussian-kernel edge-conditioned convolution of graph-neural-operator/nn_conv.py:99-194 (``NNConv_Gaussian``).

With p = edge_attr (at least 3 columns), sigma = nn(ones(1)) viewed as [C] and C = in_channels = out_channels:

    a_e   = 1 / sqrt(|p_e1 * p_e2|)
    d_ec  = a_e * exp(-p_e0^2 / sigma_c^2)
    out_n = aggr_{e: dst_e = n} x_src(e),c * d_ec  +  x_n root + bias

The reference multiplies x_j by ``diag_embed(d).view(-1, 64, 64)``, 16 KiB of fp32 per edge that autograd also keeps for
the backward.  Here d is computed inside the kernels (csrc/gauss.cu) and never stored: each application is one pass over
x and three attributes per edge, and its backward one more, which also yields the gradients of sigma and edge_attr.
"""
import ctypes

import torch
from torch.nn import Parameter

from . import _lib
from .nn_conv import (NNConv_old, _node_sets, _Pair, _f32, _ptr, _require_cuda, _require_int_channels, _stream_ptr,
                      get_plan, stats)

__all__ = ['GaussianNNConv']

MAX_CHANNELS = 4096      # csrc/plan.h kGaussMaxChannels: sigma^2 and 1 / sigma^2 are staged in shared memory


class _GaussApplyFn(torch.autograd.Function):
    """One application.  Its inputs are (x, edge_attr, sigma, root, bias, x_dst); autograd sums the sigma and edge_attr
    gradients of the T applications of a shared conv and carries sigma's into nn's parameters.  A bipartite call
    (``n_dst`` not None) takes x = x_src and the nullable x_dst; a square one passes None for both."""

    @staticmethod
    def forward(ctx, module, plan, x, edge_attr, sigma, root, bias, x_dst, n_dst):
        x32, ea32, s32 = _f32(x), _f32(edge_attr), _f32(sigma)
        ctx.pair = None if n_dst is None else _Pair(_f32(x_dst), n_dst)
        out, argmax = module._apply_impl(plan, x32, ea32, s32, ctx.pair)
        ctx.module, ctx.plan, ctx.argmax = module, plan, argmax
        ctx.dtypes = (x.dtype, edge_attr.dtype, sigma.dtype, x_dst.dtype if x_dst is not None else None)
        ctx.save_for_backward(x32, ea32, s32)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        x32, ea32, s32 = ctx.saved_tensors
        need = ctx.needs_input_grad
        dx, dea, dsig, droot, dbias, dxd = ctx.module._backward_impl(ctx.plan, x32, ea32, s32, _f32(grad_out),
                                                                     ctx.argmax, want_ea=need[3], want_sigma=need[4],
                                                                     pair=ctx.pair)
        return (None, None, dx.to(ctx.dtypes[0]) if need[2] else None,
                dea.to(ctx.dtypes[1]) if dea is not None else None,
                dsig.to(ctx.dtypes[2]) if dsig is not None else None,
                droot if need[5] else None, dbias if need[6] else None,
                dxd.to(ctx.dtypes[3]) if dxd is not None and need[7] else None, None)


class GaussianNNConv(torch.nn.Module):
    r"""graph-neural-operator/nn_conv.py:99-194 ``NNConv_Gaussian``:
    x'_i = x_i root + bias + aggr_{j in N(i)} x_j * d(e_ij), channel by channel, with
    d_c(e) = exp(-e_0^2 / sigma_c^2) / sqrt(|e_1 e_2|) and sigma = nn(ones(1)).

    Same signature, attributes, state-dict keys (``nn.*``, ``root``, ``bias``), initialisation (``reset(nn)``, then
    uniform(in) for root and bias) and repr as the reference.  ``nn`` is any module that maps a 1-element vector to C
    values; it runs in ordinary torch once per forward, so its parameters get their gradients through sigma.  ``aggr``
    in {'add', 'mean', 'max'} ('max': the rules of NNConv_old, ties to the smallest caller edge index).  Keywords:
    ``flow`` (PyG's MessagePassing kwarg) and ``precision``, accepted for symmetry with the library's other convs (and
    the NNCONV_B200_PRECISION setting of a drop-in run): the op has no GEMM, and every value computes the same fp32
    result.

    Differences from the reference: it hard-codes ``repeat(1, 64)``, so it runs only at C = 64; here any
    C = in_channels = out_channels = nn's output width up to 4096 runs, and other shapes raise NotImplementedError.
    ``edge_attr`` with fewer than 3 columns raises ValueError.  The reference's ``ones(1)`` lives on a module-global
    device; here it lives on x's device.  The rounding follows torch's fp32 order, so forward values match the
    reference's, inf and NaN included where p_e1 p_e2 = 0 or sigma_c = 0; gradients there are not finite.

    Bipartite input (PyG's form, DESIGN 4.10): ``forward(x, edge_index, edge_attr, size=None)`` also accepts ``x =
    (x_src [N_src, C], x_dst [N_dst, C] or None)`` and returns ``out[i] = x_dst[i] root + bias + aggr_{e: dst_e = i}
    x_src[src_e] * d(e)`` over N_dst rows, with NNConv_old's rules for ``size``, ``x_dst = None``, the aggregations and
    the refusals.  ``in_channels`` stays an int, and a pair raises NotImplementedError.
    """

    def __init__(self, in_channels, out_channels, nn, aggr='add', root_weight=True, bias=True, **kwargs):
        super(GaussianNNConv, self).__init__()
        self.precision = kwargs.pop('precision', None)
        self.flow = kwargs.pop('flow', 'source_to_target')
        if kwargs:
            raise TypeError('unexpected keyword arguments %s' % sorted(kwargs))
        if aggr not in ('add', 'mean', 'max'):
            raise ValueError("aggr must be 'add', 'mean' or 'max'")
        if self.flow not in _lib.FLOW:
            raise ValueError('flow must be source_to_target or target_to_source')
        if self.precision is not None and self.precision not in _lib.PREC:
            raise ValueError('precision must be one of %s' % sorted(_lib.PREC))
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
        self.reset_parameters()

    reset_parameters = NNConv_old.reset_parameters
    __repr__ = NNConv_old.__repr__
    _root_term = NNConv_old._root_term
    _root_backward = NNConv_old._root_backward

    def _sigma(self, device):
        """sigma = nn(ones(1)) as a [C] vector, after the shape checks."""
        sigma = self.nn(torch.ones(1, device=device)).reshape(-1)
        k = sigma.numel()
        if not (k == self.in_channels == self.out_channels) or k > MAX_CHANNELS:
            raise NotImplementedError(
                'GaussianNNConv: the Gaussian kernel needs nn output width == in_channels == out_channels <= %d; got nn '
                'output %d, in_channels %d, out_channels %d' % (MAX_CHANNELS, k, self.in_channels, self.out_channels))
        return sigma

    # -- reference: nn_conv.py:169-172 ---------------------------------------------------------------------------
    def forward(self, x, edge_index, edge_attr, size=None):
        x, x_dst, n_dst = _node_sets(x, size, self.flow, self.in_channels)
        pseudo = edge_attr.unsqueeze(-1) if edge_attr.dim() == 1 else edge_attr
        sigma = self._sigma(x.device)
        if pseudo.dim() != 2 or pseudo.size(1) < 3:
            raise ValueError('GaussianNNConv: edge_attr needs at least 3 columns (p0 for the Gaussian, p1 * p2 for its '
                             'amplitude); got shape %s' % (tuple(pseudo.shape),))
        NNConv_old._check_inputs(self, x, edge_index, pseudo)
        _require_cuda(sigma, 'nn(ones(1))')
        with torch.cuda.device(x.device):
            plan = get_plan(edge_index, x.size(0) if n_dst is None else (x.size(0), n_dst), self.flow)
            needs_grad = torch.is_grad_enabled() and (
                x.requires_grad or pseudo.requires_grad or sigma.requires_grad or
                any(p is not None and p.requires_grad for p in (self.root, self.bias)) or
                (x_dst is not None and x_dst.requires_grad))
            if not needs_grad:
                pair = None if n_dst is None else _Pair(_f32(x_dst), n_dst)
                return self._apply_impl(plan, _f32(x), _f32(pseudo), _f32(sigma), pair)[0]
            return _GaussApplyFn.apply(self, plan, x, pseudo, sigma, self.root, self.bias, x_dst, n_dst)

    # -- library calls ---------------------------------------------------------------------------------------------
    def _apply_impl(self, plan, x32, ea32, s32, pair=None):
        """One application (nnconv_gauss_apply); returns (out, argmax), argmax None unless aggr='max'.  A bipartite
        call (pair: the _Pair of x_dst) runs the messages from x32 = x_src with no root or bias, then adds x_dst root +
        bias (nnconv_root_term); out has N_dst rows."""
        L = _lib.lib()
        dev = x32.device
        aggr = _lib.AGGR[self.aggr]
        C = self.out_channels
        ws_b = ctypes.c_size_t()
        _lib.check(L.nnconv_gauss_apply_sizes(plan.handle, C, aggr, ctypes.byref(ws_b)))
        ws = torch.empty(ws_b.value, dtype=torch.uint8, device=dev)
        out = torch.empty(plan.N_dst, C, dtype=torch.float32, device=dev)
        argmax = torch.empty(plan.N_dst, C, dtype=torch.int32, device=dev) if self.aggr == 'max' else None
        root, bias = (_f32(self.root), _f32(self.bias)) if pair is None else (None, None)
        n_l = ctypes.c_int64(0)
        _lib.check(L.nnconv_gauss_apply(plan.handle, _ptr(ea32), ea32.size(1), _ptr(s32), C, _ptr(x32), _ptr(root),
                                        _ptr(bias), aggr, _ptr(out), _ptr(argmax), _ptr(ws), ws_b.value,
                                        _stream_ptr(dev), ctypes.byref(n_l)))
        stats['launches'] += n_l.value
        if pair is not None:
            self._root_term(pair, out)
        stats['applies'] += 1
        return out, argmax

    def _backward_impl(self, plan, x32, ea32, s32, g32, argmax, want_ea, want_sigma, pair=None):
        """dx, d edge_attr (None unless want_ea), dsigma (None unless want_sigma), droot, dbias, dx_dst of one
        application.  A bipartite call (pair) takes droot, dbias and dx_dst from the root term's backward, else dx_dst
        is None."""
        L = _lib.lib()
        dev = x32.device
        with torch.cuda.device(dev):
            square = pair is None
            dx = torch.empty_like(x32)
            dea = torch.empty_like(ea32) if want_ea else None
            dsig = torch.empty_like(s32) if want_sigma else None
            droot = torch.empty_like(self.root, dtype=torch.float32) if self.root is not None and square else None
            dbias = torch.empty_like(self.bias, dtype=torch.float32) if self.bias is not None and square else None
            root = _f32(self.root) if square else None
            n_l = ctypes.c_int64(0)
            _lib.check(L.nnconv_gauss_backward(plan.handle, _ptr(ea32), ea32.size(1), _ptr(s32), self.out_channels,
                                               _ptr(x32), _ptr(root), _lib.AGGR[self.aggr], _ptr(argmax), _ptr(g32),
                                               _ptr(dx), _ptr(droot), _ptr(dbias), _ptr(dsig), _ptr(dea),
                                               _stream_ptr(dev), ctypes.byref(n_l)))
            stats['launches'] += n_l.value
            dxd = None
            if not square:
                dxd, droot, dbias = self._root_backward(pair, g32)
            stats['backwards'] += 1
        return dx, dea, dsig, droot, dbias, dxd
