"""Exact integer probes of the Gaussian-kernel NNConv.

p_e0 = 0, so exp(-p0^2 / sigma^2) = 1 for every sigma; p_e1 = +-2^i and p_e2 = +-2^j with i + j even, so |p1 p2| is a
power of four and a_e = 1 / sqrt(|p1 p2|) a power of two in [1/4, 4].  x, the output gradient, root, bias and the
weights of nn (which give a sigma of small nonzero integers) are small integers.  Every message x * a is then a
multiple of 1/4 below 2^5, every sum of the forward and the backward stays far below 2^22, and the edge_attr gradients
-(sum_c u) / (2 p) divide by powers of two: no operation rounds, in any order, so the library must equal the fp64 oracle
bit for bit.  tests/test_gauss_host.py proves that budget on the CPU by comparing an fp32 evaluation with the fp64 one.
"""
import torch

from tests import gauss_oracle as G


def graph(n=300, e=6000, seed=0):
    """Random graph with a hub source (node 0: 1/6 of the edges, > 128 so it spans many tiles), nodes 0..4 without
    in-edges, nodes n-5..n-1 without out-edges (beside the hub) and duplicate edges."""
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n - 5, (e,), generator=g)
    dst = torch.randint(5, n, (e,), generator=g)
    src[: e // 6] = 0
    src[10:20], dst[10:20] = src[9], dst[9]
    perm = torch.randperm(e, generator=g)
    return torch.stack([src[perm], dst[perm]])


def edge_attr(e, k_in=3, seed=0):
    """[e, k_in]: p0 = 0, p1 p2 a power of four, the other columns small integers (unused by the op)."""
    g = torch.Generator().manual_seed(seed)
    ea = torch.randint(-3, 4, (e, k_in), generator=g).double()
    i = torch.randint(-2, 3, (e,), generator=g)
    j = torch.randint(-1, 2, (e,), generator=g) * 2 - (i % 2)          # i + j even, j in [-3, 2]
    s1 = torch.where(torch.rand(e, generator=g) < 0.5, -1.0, 1.0).double()
    s2 = torch.where(torch.rand(e, generator=g) < 0.5, -1.0, 1.0).double()
    ea[:, 0] = 0
    ea[:, 1] = s1 * torch.pow(2.0, i.double())
    ea[:, 2] = s2 * torch.pow(2.0, j.double())
    return ea


def nn_module(c, seed=0):
    """Linear(1, c) whose output on ones(1) is a vector of nonzero integers in [-4, 4]."""
    g = torch.Generator().manual_seed(seed)
    lin = torch.nn.Linear(1, c)
    w = torch.randint(-2, 3, (c, 1), generator=g).double()
    b = torch.randint(1, 3, (c,), generator=g).double() * torch.where(torch.rand(c, generator=g) < 0.5, -1.0, 1.0)
    b = torch.where(w[:, 0] + b == 0, b + b, b)
    with torch.no_grad():
        lin.weight.copy_(w)
        lin.bias.copy_(b)
    return lin


def tensors(n, c, seed=0):
    """x [n, c], gout [n, c], root [c, c], bias [c]: small integers (fp64)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-4, 5, (n, c), generator=g).double()
    gout = torch.randint(-3, 4, (n, c), generator=g).double()
    root = torch.randint(-1, 2, (c, c), generator=g).double()
    bias = torch.randint(-2, 3, (c,), generator=g).double()
    return x, gout, root, bias


def reference(x, ei, ea, lin, root, bias, gout, aggr, dtype=torch.float64, flow='source_to_target', n_apps=1):
    """out and the gradients of sum(out * gout) w.r.t. x, edge_attr, nn's weight and bias, root and bias, with the
    oracle evaluated in `dtype`.  n_apps > 1 applies one conv n_apps times to the same x (out = the sum of them, so the
    gradients are sums over the applications)."""
    xs = x.detach().to(dtype).requires_grad_()
    eas = ea.detach().to(dtype).requires_grad_()
    w = lin.weight.detach().to(dtype).requires_grad_()
    b = lin.bias.detach().to(dtype).requires_grad_()
    r = root.detach().to(dtype).requires_grad_() if root is not None else None
    bb = bias.detach().to(dtype).requires_grad_() if bias is not None else None
    out = 0
    argmaxes = []
    for _ in range(n_apps):
        sigma = torch.ones(1, dtype=dtype) @ w.t() + b
        o, am = G.gauss_forward(xs, ei, eas, sigma, r, bb, aggr, flow)
        out = out + o
        argmaxes.append(am)
    (out * gout.to(dtype)).sum().backward()
    grads = {'x': xs.grad, 'edge_attr': eas.grad, 'nn.weight': w.grad, 'nn.bias': b.grad}
    if r is not None:
        grads['root'] = r.grad
    if bb is not None:
        grads['bias'] = bb.grad
    return out.detach(), argmaxes[0], grads
