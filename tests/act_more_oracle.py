"""fp64 reference of an edge network whose hidden activation is Hardtanh, ReLU6, Hardsigmoid, SELU, CELU, Softsign or
LogSigmoid, and of NNConv / DiagNNConv over it.

The activations are applied as torch's own modules in fp64, so a gradient taken through this restatement is torch's
derivative, including its choice at the kinks of the clamps (0 at a bound).  The convolutions are tests/act_oracle.py's:
the hidden layers are evaluated here and handed to it as the input of a single-Linear network.
"""
import torch

from tests import act_oracle as A

# kind -> a torch module with that activation, p its parameter (None, Hardtanh's (lo, hi) or CELU's alpha)
MODULES = {
    'relu6': lambda p: torch.nn.ReLU6(),
    'hardtanh': lambda p: torch.nn.Hardtanh(*p),
    'hardsigmoid': lambda p: torch.nn.Hardsigmoid(),
    'selu': lambda p: torch.nn.SELU(),
    'celu': lambda p: torch.nn.CELU(p),
    'softsign': lambda p: torch.nn.Softsign(),
    'logsigmoid': lambda p: torch.nn.LogSigmoid(),
}

_L, _AL = 1.0507009873554805, 1.6732632423543772


def _inside(y, lo, hi, a):
    return torch.where((y > lo) & (y < hi), torch.full_like(y, a), torch.zeros_like(y))


# kind -> f'(z) from the output y = f(z), as the library computes it (torch's backward at the bounds and at 0)
GRADS = {
    'relu6': lambda y, p: _inside(y, 0.0, 6.0, 1.0),
    'hardtanh': lambda y, p: _inside(y, p[0], p[1], 1.0),
    'hardsigmoid': lambda y, p: _inside(y, 0.0, 1.0, 1.0 / 6.0),
    'selu': lambda y, p: torch.where(y > 0, torch.full_like(y, _L), y + _L * _AL),
    'celu': lambda y, p: torch.where(y > 0, torch.ones_like(y), y / p + 1),
    'softsign': lambda y, p: (1 - y.abs()) ** 2,
    'logsigmoid': lambda y, p: -torch.expm1(y),
}

# the spec the library reads from each module (graph_pde_b200.nn_conv._act_spec)
SPECS = {
    'relu6': lambda p: ('clamp', (1.0, 0.0, 0.0, 6.0)),
    'hardtanh': lambda p: ('clamp', (1.0, 0.0, float(p[0]), float(p[1]))),
    'hardsigmoid': lambda p: ('clamp', (1.0 / 6.0, 0.5, 0.0, 1.0)),
    'selu': lambda p: ('scaled_elu', (_L, _AL, 1.0)),
    'celu': lambda p: ('scaled_elu', (1.0, float(p), 1.0 / float(p))),
    'softsign': lambda p: ('softsign', ()),
    'logsigmoid': lambda p: ('logsigmoid', ()),
}


def hidden(edge_attr, weights, biases, act, p):
    """The edge network up to its last Linear: Linear -> f -> ... -> Linear -> f."""
    f = MODULES[act](p)
    h = edge_attr
    for w, b in zip(weights, biases):
        h = f(torch.nn.functional.linear(h, w, b))
    return h


def nnconv_forward(x, edge_index, edge_attr, weights, biases, root=None, bias=None, aggr='add', act='relu6', p=None,
                   **kw):
    """(out, argmax) of NNConv_old with this edge network (tests/act_oracle.nnconv_forward)."""
    h = hidden(edge_attr, weights[:-1], biases[:-1], act, p)
    return A.nnconv_forward(x, edge_index, h, weights[-1:], biases[-1:], root, bias, aggr, **kw)


def diag_forward(x, edge_index, edge_attr, weights, biases, root=None, bias=None, aggr='add', act='relu6', p=None):
    h = hidden(edge_attr, weights[:-1], biases[:-1], act, p)
    return A.diag_forward(x, edge_index, h, weights[-1:], biases[-1:], root, bias, aggr)
