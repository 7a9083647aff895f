"""fp64 reference of an edge network with another hidden activation than ReLU, and of NNConv / DiagNNConv over it.

DenseNet(layers, nonlinearity) (graph-neural-operator/utilities.py:201-227) puts one ``nonlinearity()`` after every
Linear but the last.  ``ACTS`` restates the five activations the library runs with torch's semantics; the NNConv
restatement is oracle/nnconv_oracle.py's with this edge network in place of the ReLU one (add and mean), and
tests/diag_oracle.py's for the diagonal kernel.
"""
import torch
import torch.nn.functional as F

from tests import max_oracle as M

# kind -> f(z, p), with p the LeakyReLU slope / ELU alpha
ACTS = {
    'relu': lambda z, p: torch.relu(z),
    'leaky_relu': lambda z, p: torch.where(z > 0, z, p * z),
    'elu': lambda z, p: torch.where(z > 0, z, p * torch.expm1(z)),
    'tanh': lambda z, p: torch.tanh(z),
    'sigmoid': lambda z, p: torch.sigmoid(z),
}

# kind -> f'(z) from the output y = f(z) (what the library's backward computes; torch's own backward at y = 0)
GRADS = {
    'relu': lambda y, p: (y > 0).to(y.dtype),
    'leaky_relu': lambda y, p: torch.where(y > 0, torch.ones_like(y), torch.full_like(y, p)),
    'elu': lambda y, p: torch.where(y > 0, torch.ones_like(y), y + p),
    'tanh': lambda y, p: 1 - y * y,
    'sigmoid': lambda y, p: y * (1 - y),
}

# kind -> a torch module with that activation (for DenseNet(layers, nonlinearity))
MODULES = {
    'relu': lambda p: torch.nn.ReLU(),
    'leaky_relu': lambda p: torch.nn.LeakyReLU(p),
    'elu': lambda p: torch.nn.ELU(p),
    'tanh': lambda p: torch.nn.Tanh(),
    'sigmoid': lambda p: torch.nn.Sigmoid(),
}


def dense_net(edge_attr, weights, biases, act='relu', p=0.0):
    """Linear -> f -> ... -> Linear, f after every layer but the last."""
    h = edge_attr
    n = len(weights)
    for l in range(n):
        h = F.linear(h, weights[l], biases[l])
        if l != n - 1:
            h = ACTS[act](h, p)
    return h


def nnconv_forward(x, edge_index, edge_attr, weights, biases, root=None, bias=None, aggr='add', act='relu', p=0.0,
                   flow='source_to_target', argmax=None):
    """(out, argmax) of NNConv_old (graph-neural-operator/nn_conv.py:267-282) with this edge network; argmax is None
    unless aggr == 'max' (given: route the max by it)."""
    x = x.unsqueeze(-1) if x.dim() == 1 else x
    pseudo = edge_attr.unsqueeze(-1) if edge_attr.dim() == 1 else edge_attr
    src, dst = (edge_index[1], edge_index[0]) if flow == 'target_to_source' else (edge_index[0], edge_index[1])
    n, cin = x.size(0), x.size(1)
    cout = weights[-1].size(0) // cin
    w = dense_net(pseudo, weights, biases, act, p).view(-1, cin, cout)
    msg = torch.matmul(x[src].unsqueeze(1), w).squeeze(1)
    if aggr == 'max':
        if argmax is None:
            argmax = M.winners(msg, dst, n)
        out = M.max_term(msg, argmax)
    else:
        out = torch.zeros(n, cout, dtype=msg.dtype).index_add(0, dst, msg)
        if aggr == 'mean':
            cnt = torch.zeros(n, dtype=msg.dtype).index_add(0, dst, torch.ones(dst.numel(), dtype=msg.dtype))
            out = out / cnt.clamp(min=1).unsqueeze(-1)
    if root is not None:
        out = out + x @ root
    if bias is not None:
        out = out + bias
    return out, argmax


def diag_forward(x, edge_index, edge_attr, weights, biases, root=None, bias=None, aggr='add', act='relu', p=0.0):
    """The diagonal-kernel conv (graph-neural-operator/nn_conv.py:73-93): x_src * nn(edge_attr) per channel."""
    src, dst = edge_index[0], edge_index[1]
    n = x.size(0)
    msg = x[src] * dense_net(edge_attr, weights, biases, act, p)
    if aggr == 'max':
        out = M.max_term(msg, M.winners(msg, dst, n))
    else:
        out = torch.zeros(n, msg.size(1), dtype=msg.dtype).index_add(0, dst, msg)
        if aggr == 'mean':
            cnt = torch.zeros(n, dtype=msg.dtype).index_add(0, dst, torch.ones(dst.numel(), dtype=msg.dtype))
            out = out / cnt.clamp(min=1).unsqueeze(-1)
    if root is not None:
        out = out + x @ root
    if bias is not None:
        out = out + bias
    return out
