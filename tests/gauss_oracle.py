"""fp64 reference of the Gaussian-kernel NNConv (graph-neural-operator/nn_conv.py:99-194, class NNConv_Gaussian there).

The reference multiplies x_j by diag_embed(d_e).view(-1, C, C) with d_ec = exp(-p_e0^2 / sigma_c^2) / sqrt(|p_e1 p_e2|)
and sigma = nn(ones(1)); that is x_j * d_e channel by channel.  Aggregation as PyG's MessagePassing: add, mean (the
empty mean is 0) or max (tests/max_oracle.py: ties to the smallest caller edge index, 0 and argmax -1 without in-edges).
Differentiable w.r.t. x, edge_attr, sigma, root and bias.
"""
import torch

from tests import max_oracle as M


def diagonal(edge_attr, sigma):
    """d [E, C] in the caller's edge order, in the reference's order of operations (nn_conv.py:176-179)."""
    p = edge_attr
    a = 1 / torch.sqrt(torch.abs(p[:, 1] * p[:, 2]))
    b = torch.exp(-1 * (p[:, 0] ** 2).view(-1, 1) / (sigma ** 2).view(1, -1))
    return a.reshape(-1, 1) * b


def gauss_forward(x, edge_index, edge_attr, sigma, root=None, bias=None, aggr='add', flow='source_to_target',
                  argmax=None):
    """(out, argmax) of one application; argmax is None unless aggr == 'max' (given: route the max by it)."""
    x = x.unsqueeze(-1) if x.dim() == 1 else x
    pseudo = edge_attr.unsqueeze(-1) if edge_attr.dim() == 1 else edge_attr
    src, dst = (edge_index[1], edge_index[0]) if flow == 'target_to_source' else (edge_index[0], edge_index[1])
    n = x.size(0)
    msg = x[src] * diagonal(pseudo, sigma.reshape(-1))
    if aggr == 'max':
        if argmax is None:
            argmax = M.winners(msg, dst, n)
        out = M.max_term(msg, argmax)
    else:
        out = torch.zeros(n, msg.size(1), dtype=msg.dtype).index_add(0, dst, msg)
        if aggr == 'mean':
            cnt = torch.zeros(n, dtype=msg.dtype).index_add(0, dst, torch.ones(dst.numel(), dtype=msg.dtype))
            out = out / cnt.clamp(min=1).unsqueeze(-1)
    if root is not None:
        out = out + x @ root
    if bias is not None:
        out = out + bias
    return out, argmax
