"""fp64 reference of GCNConv (PyG 1.x ``gcn_norm`` + ``propagate`` restated with index_add; DESIGN 4.8).

Self loops as ``add_remaining_self_loops``: the caller's loops leave the edge list and every node gets one loop of weight
1 if it had one, else ``fill`` (2 when improved).  Without added loops (``add_self_loops=False``) or without
normalisation the caller's list is used as it is, loops included, every edge of weight 1.  Degrees are summed at the
target; deg^-1/2 of a zero degree is 0.  out = sum_e norm_e (x W)[src_e] + bias, x W first as PyG computes it.
"""
import math

import torch


def gcn_norm(edge_index, n, improved=False, add_self_loops=True, normalize=True, flow='source_to_target',
             dtype=torch.float64):
    """(src, dst, norm) of every term of A_hat, the loops as explicit entries."""
    row0, row1 = edge_index[0].long(), edge_index[1].long()
    src, dst = (row0, row1) if flow == 'source_to_target' else (row1, row0)
    dev = src.device
    if not normalize:
        return src, dst, torch.ones(src.numel(), dtype=dtype, device=dev)
    w = torch.ones(src.numel(), dtype=dtype, device=dev)
    if add_self_loops:
        keep = src != dst
        loop_w = torch.full((n,), 2.0 if improved else 1.0, dtype=dtype, device=dev)
        loop_w[src[~keep]] = 1.0
        nodes = torch.arange(n, device=dev)
        src = torch.cat([src[keep], nodes])
        dst = torch.cat([dst[keep], nodes])
        w = torch.cat([w[keep], loop_w])
    deg = torch.zeros(n, dtype=dtype, device=dev).index_add_(0, dst, w)
    dinv = deg.pow(-0.5)
    dinv[torch.isinf(dinv)] = 0
    return src, dst, dinv[src] * w * dinv[dst]


def gcn_forward(x, edge_index, weight, bias=None, improved=False, add_self_loops=True, normalize=True,
                flow='source_to_target', dtype=torch.float64):
    """One application in ``dtype`` (differentiable w.r.t. x, weight and bias)."""
    n = x.size(0)
    src, dst, norm = gcn_norm(edge_index, n, improved, add_self_loops, normalize, flow, dtype)
    xw = x.to(dtype) @ weight.to(dtype)
    out = torch.zeros(n, xw.size(1), dtype=dtype, device=x.device).index_add_(0, dst, norm[:, None] * xw[src])
    return out + bias.to(dtype) if bias is not None else out


class GCNConv(torch.nn.Module):
    """The PyG 1.x module restated over gcn_forward: same signature, parameters, init stream and repr as PyG's."""

    def __init__(self, in_channels, out_channels, improved=False, cached=False, add_self_loops=True, normalize=True,
                 bias=True, **kwargs):
        super(GCNConv, self).__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.improved, self.add_self_loops, self.normalize = improved, add_self_loops, normalize
        self.weight = torch.nn.Parameter(torch.Tensor(in_channels, out_channels))
        self.bias = torch.nn.Parameter(torch.Tensor(out_channels)) if bias else None
        stdv = math.sqrt(6.0 / (in_channels + out_channels))
        self.weight.data.uniform_(-stdv, stdv)
        if self.bias is not None:
            self.bias.data.fill_(0)

    def forward(self, x, edge_index, edge_weight=None):
        assert edge_weight is None
        return gcn_forward(x, edge_index, self.weight, self.bias, self.improved, self.add_self_loops, self.normalize,
                           dtype=x.dtype)

    def __repr__(self):
        return '{}({}, {})'.format(self.__class__.__name__, self.in_channels, self.out_channels)
