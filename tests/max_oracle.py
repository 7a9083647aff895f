"""fp64 reference of NNConv aggr='max', written independently of the library's packed keys.

Per node n and channel o:  out[n, o] = max_{e: dst_e = n} m_e[o] + (x root + bias)[n, o],  m_e = x_src . K_e the
message of aggr='add'.  A node without in-edges gets 0 for the max term and argmax -1.  Ties go to the smallest index
in the caller's edge_index; -0 equals +0; a NaN message wins (among NaN messages the smallest index).  The max is
taken in three steps: scatter_reduce('amax') of the values, the smallest caller index among the edges equal to that
max (scatter_reduce('amin')), and a gather of the winning messages -- so autograd routes each gradient entry to the
winning edge alone.
"""
import torch

from oracle import nnconv_oracle as O


def messages(x, src, edge_attr, weights, biases, cin, cout, edge_chunk=None):
    """m_e [E, cout] in the caller's edge order (edge_chunk: the edge network in chunks of that many edges)."""
    e = src.numel()
    step = e if not edge_chunk else edge_chunk
    parts = []
    for s in range(0, e, max(step, 1)):
        k = O.dense_net(edge_attr[s:s + step], weights, biases).view(-1, cin, cout)
        parts.append(torch.bmm(x[src[s:s + step]].unsqueeze(1), k).squeeze(1))
    return torch.cat(parts) if parts else x.new_zeros(0, cout)


def winners(msg, dst, n_nodes):
    """argmax [n_nodes, cout] int64: the caller index of the winning edge of every (node, channel), -1 when empty."""
    v = msg.detach()
    e, cout = v.shape
    idx = dst.view(-1, 1).expand(e, cout)
    nan = torch.isnan(v)
    vals = torch.where(nan, torch.full_like(v, float('inf')), v)
    # 1. the max of the values (a NaN counted as above +inf through its own flag)
    mx = v.new_full((n_nodes, cout), float('-inf')).scatter_reduce(0, idx, vals, 'amax', include_self=False)
    any_nan = v.new_zeros(n_nodes, cout).scatter_reduce(0, idx, nan.to(v.dtype), 'amax', include_self=False) > 0
    win = torch.where(any_nan[dst], nan, (vals == mx[dst]) & ~nan)
    # 2. the smallest caller index among the edges equal to it
    eidx = torch.arange(e, dtype=v.dtype, device=v.device).view(-1, 1).expand(e, cout)
    cand = torch.where(win, eidx, torch.full_like(eidx, float(e)))
    first = v.new_full((n_nodes, cout), float(e)).scatter_reduce(0, idx, cand, 'amin', include_self=True)
    am = first.to(torch.int64)
    am[am == e] = -1
    return am


def max_term(msg, argmax):
    """3. the gather of the winning messages (0 where argmax is -1): differentiable w.r.t. msg."""
    safe = argmax.clamp(min=0)
    g = msg.gather(0, safe)
    return torch.where(argmax >= 0, g, torch.zeros_like(g))


def nnconv_forward_max(x, edge_index, edge_attr, weights, biases, root=None, bias=None, edge_chunk=None,
                       argmax=None):
    """(out, argmax) of one aggr='max' application; argmax given: route by it instead of computing it (the
    oracle's backward given the library's argmax)."""
    cin, n = x.size(1), x.size(0)
    cout = weights[-1].size(0) // cin
    src, dst = edge_index[0], edge_index[1]
    msg = messages(x, src, edge_attr, weights, biases, cin, cout, edge_chunk)
    if argmax is None:
        argmax = winners(msg, dst, n)
    out = max_term(msg, argmax)
    if root is not None:
        out = out + x @ root
    if bias is not None:
        out = out + bias
    return out, argmax


def win_share(argmax, n_edges):
    """Share of the edges that win at least one (node, channel)."""
    a = argmax[argmax >= 0].unique()
    return a.numel() / max(n_edges, 1)
