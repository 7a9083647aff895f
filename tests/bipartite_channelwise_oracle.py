"""fp64 restatement of the bipartite channel-wise convs (DESIGN 4.10), differentiable with autograd:

    out[i] = x_dst[i] root + bias + aggr_{e: dst_e = i} x_src[src_e] * d_e

over N_dst target rows; edge_index row 0 indexes x_src, row 1 x_dst.  d [E, C] is the diagonal in the caller's edge
order: ``diag_d`` for DiagNNConv (d_e = nn(e)), ``gauss_d`` for GaussianNNConv.  aggr 'add', 'mean' (in-degree over the
targets, 1/max(deg, 1)) or 'max' (tests/max_oracle.py: per channel, ties to the smallest caller edge, 0 and argmax -1
for a target without in-edges).  x_dst None drops the root term."""
import torch

from oracle import nnconv_oracle as O
from tests import gauss_oracle as G
from tests import max_oracle as M


def diag_d(edge_attr, weights, biases):
    return O.dense_net(edge_attr, weights, biases)


def gauss_d(edge_attr, sigma):
    return G.diagonal(edge_attr, sigma.reshape(-1))


def forward(x_src, x_dst, edge_index, d, root, bias, aggr, n_dst, argmax=None):
    """(out, argmax) of one application; argmax is None unless aggr == 'max' (given: route the max by it)."""
    src, dst = edge_index[0].long(), edge_index[1].long()
    msg = x_src[src] * d
    if aggr == 'max':
        if argmax is None:
            argmax = M.winners(msg, dst, n_dst)
        out = M.max_term(msg, argmax)
    else:
        out = torch.zeros(n_dst, msg.size(1), dtype=msg.dtype, device=msg.device).index_add(0, dst, msg)
        if aggr == 'mean':
            deg = torch.bincount(dst, minlength=n_dst).clamp(min=1).to(msg.dtype)
            out = out / deg.unsqueeze(1)
    if x_dst is not None and root is not None:
        out = out + x_dst @ root
    if bias is not None:
        out = out + bias
    return out, argmax
