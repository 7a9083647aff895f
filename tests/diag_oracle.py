"""fp64 reference of the diagonal-kernel NNConv (graph-neural-operator/nn_conv.py:73-93, class NNConv there).

The reference forms diag_embed(nn(e)).view(-1, in, out) and multiplies x_j by it; with nn's output width == in == out
that is x_j * k_e channel by channel, k_e = nn(e).  Aggregation as PyG's MessagePassing: add, mean (the empty mean is
0) or max (tests/max_oracle.py: ties to the smallest caller edge index, 0 and argmax -1 without in-edges).
"""
import torch

from oracle import nnconv_oracle as O
from tests import max_oracle as M


def messages(x, src, edge_attr, weights, biases):
    """m_e = x[src_e] * nn(edge_attr_e)  [E, out] in the caller's edge order."""
    return x[src] * O.dense_net(edge_attr, weights, biases)


def nnconv_diag_forward(x, edge_index, edge_attr, weights, biases, root=None, bias=None, aggr='add', flow='source_to_target',
                        argmax=None):
    """(out, argmax) of one application; argmax is None unless aggr == 'max' (given: route the max by it)."""
    x = x.unsqueeze(-1) if x.dim() == 1 else x                                   # nn_conv.py:82
    pseudo = edge_attr.unsqueeze(-1) if edge_attr.dim() == 1 else edge_attr      # nn_conv.py:83
    src, dst = (edge_index[1], edge_index[0]) if flow == 'target_to_source' else (edge_index[0], edge_index[1])
    n = x.size(0)
    msg = messages(x, src, pseudo, weights, biases)
    if aggr == 'max':
        if argmax is None:
            argmax = M.winners(msg, dst, n)
        out = M.max_term(msg, argmax)
    else:
        out = torch.zeros(n, msg.size(1), dtype=msg.dtype).index_add(0, dst, msg)
        if aggr == 'mean':
            cnt = torch.zeros(n, dtype=msg.dtype).index_add(0, dst, torch.ones(dst.numel(), dtype=msg.dtype))
            out = out / cnt.clamp(min=1).unsqueeze(-1)
    if root is not None:                                                         # nn_conv.py:89-90
        out = out + x @ root
    if bias is not None:                                                         # nn_conv.py:91-92
        out = out + bias
    return out, argmax
