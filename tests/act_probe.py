"""An exact integer probe of an edge network with LeakyReLU(0.25) between its layers (tests/probes.py builds the graph,
the sparse {-1, 0, +1} weights and the integer inputs; this module proves the budget for the other activation).

Every hidden unit is ``f(h_a - h_b + bias)`` with a small integer bias, so pre-activations take both signs; with slope
1/4 a negative one becomes a multiple of 1/4 after layer 1 and of 1/16 after layer 2, still a few significant bits.
The backward multiplies by f'(y) in {1, 1/4}, again a power of two.  ``assert_exact`` proves, in fp64 on the CPU, that
every 16-bit buffer of the forward and of the tensor-core backward stores its values unchanged and that every fp32 sum
stays within 2^22 quanta (probes.py's budget), so the library must equal fp64 autograd bit for bit.  It follows
probes.assert_exact (aggr='add', formulation C and B) with the activation and its derivative in place of ReLU and its
mask, and with the quanta of the hidden layers taken from their dyadic activations.
"""
import torch

from tests import act_oracle as A
from tests import probes as P

SLOPE = 0.25
LAYERS = [3, 64, 64, 64 * 64]      # two hidden layers of LeakyReLU, in = out = 64 (the tensor-core backward's shape)


def make(ei, n_nodes, seed=3, T=2, grad=True, precision='f16'):
    """The probe (a probes.Probe) on graph ``ei``.  Its x stays small integers at every precision: the 1/16 quanta of h
    leave no room for 12-bit inputs in the node sums.  bf16 keeps 8 significant bits, so output-gradient rows are
    non-zero at 1/32 of the nodes only (the hub's dY sums over 300 edges)."""
    return P.make_probe(ei, n_nodes, LAYERS, 64, 64, seed=seed, T=T, grad=grad,
                        g_rows=1 / 32. if precision == 'bf16' else 1.0)


def graph():
    """A 600-node graph with a hub source of 300 out-edges, duplicated edges, self-loops and nodes without in-edges."""
    return P.mixed_graph(n_nodes=600, n_edges=6000, hub=300, seed=11), 600


def hidden(ea, ws, bs):
    """[h_0 = ea, h_1, ..., h_{L-1}] with the LeakyReLU, and the pre-activations [z_1, ..., z_{L-1}], fp64."""
    hs, zs = [ea.double()], []
    for w, b in zip(ws[:-1], bs[:-1]):
        zs.append(hs[-1] @ w.t() + b)
        hs.append(A.ACTS['leaky_relu'](zs[-1], SLOPE))
    return hs, zs


def _grad(y):
    return A.GRADS['leaky_relu'](y, SLOPE)


def assert_exact(p, precision):
    """Raise probes.NotExact unless the forward (formulation C and, at f16 / bf16, B) and the backward of ``p`` are
    computed without rounding at ``precision``.  Returns the pre-activations of the distinct edge-attribute rows."""
    ws, bs = p.ws, p.bs
    ea = p.ea.double().cpu()
    src, dst = (t.cpu() for t in p.src_dst())
    for l, (w, b) in enumerate(zip(ws, bs)):
        P.check_16bit('weight %d' % l, w, precision)
        P.check_16bit('bias %d' % l, b, precision)
    uniq, inv = P._distinct_rows(ea)
    hs, zs = hidden(uniq, ws, bs)
    w1, b1 = ws[0], bs[0]
    hi, lo = P._split(uniq, 'bf16' if precision == 'bf16' else 'f16')
    if precision != 'fp32':
        P.check_16bit('A1 hi(edge_attr)', hi, precision)
        P.check_16bit('A1 lo(edge_attr)', lo, precision)
    P.check_sum('first layer', (hi.abs() + lo.abs()) @ w1.abs().t() + b1.abs(), P._lowest_bit(uniq) * P._lowest_bit(w1))
    n_lin = len(ws)
    for l in range(1, n_lin):
        P.check_16bit('hidden activation %d' % l, hs[l], precision)
        if l >= 2:
            P.check_sum('hidden layer %d' % l, hs[l - 1].abs() @ ws[l - 1].abs().t() + bs[l - 1].abs(),
                        P._lowest_bit(hs[l - 1]) * P._lowest_bit(ws[l - 1]))
            P.check_product('hidden layer %d' % l, hs[l - 1], ws[l - 1], precision)
    h, wl, bl = hs[-1], ws[-1], bs[-1]
    cin, cout = p.cin, p.cout
    wl3 = wl.view(cin, cout, -1)
    if int((wl3 != 0).sum(0).max()) > 1:
        raise P.NotExact('W_L: a (channel, hidden unit) column reads more than one input channel')
    xq = min(P._lowest_bit(x) for x in p.x)
    xmax = torch.stack([x.abs().max(1).values for x in p.x]).max(0).values
    for t, x in enumerate(p.x):
        P.check_16bit('Xc, input %d' % t, x / torch.tensor(
            [P._pow2_ge(float(v)) for v in x.abs().max(1).values]).unsqueeze(1), precision)
        P.check_16bit('Y, input %d' % t, x, precision, normalise=True)
    P.check_product('contraction h . Y', h, torch.cat(p.x), precision)
    quantum = P._lowest_bit(h) * P._lowest_bit(wl) * xq
    per_code = h.abs() @ wl3.abs().sum(0).t() + bl.abs().view(cin, cout).sum(0)
    msg = per_code.max(1).values[inv] * xmax[src]
    P.check_sum('message', msg, quantum)
    init = xmax * p.root.abs().sum(0).max() + p.bias.abs().max()
    P.check_sum('scatter into out[dst]', init.index_add(0, dst, msg), quantum)
    if precision in ('f16', 'bf16'):
        P.check_16bit('K_e (formulation B)', h @ wl.t() + bl, precision)
        P.check_sum('K_e build', h.abs() @ wl.abs().t() + bl.abs(), P._lowest_bit(h))
    if p.grad_out is not None:
        _backward(p, precision, src, dst, inv, hs)
    return zs


def _backward(p, precision, src, dst, inv, hs_u):
    """probes._assert_exact_backward (aggr='add') with dz = dh * f'(h) in place of the ReLU mask."""
    ws = p.ws
    cin, cout = p.cin, p.cout
    hs = [a[inv] for a in hs_u]
    h, wl = hs[-1], ws[-1]
    gq = min(P._lowest_bit(g) for g in p.grad_out)
    wl3 = wl.view(cin, cout, -1).abs()
    order = torch.argsort(src, stable=True)
    counts = torch.bincount(src, minlength=p.n_nodes)
    starts = torch.cumsum(counts, 0) - counts
    for t, (x, g) in enumerate(zip(p.x, p.grad_out)):
        G = g[dst]
        P.check_16bit('G, application %d' % t, G, precision, normalise=True)
        P.check_product('k_dy h . G', h, G, precision)
        dwl_abs = torch.zeros_like(wl3)
        for c in torch.nonzero(counts).flatten().tolist():
            rows = order[int(starts[c]):int(starts[c] + counts[c])]
            dY, dyabs = h[rows].t() @ G[rows], h[rows].abs().t() @ G[rows].abs()
            P.check_sum('dY, application %d' % t, dyabs, P._lowest_bit(h) * gq)
            P.check_16bit('dY, application %d' % t, dY, precision, normalise=True)
            P.check_sum('dx = dY : W_L, application %d' % t, torch.einsum('ko,iok->i', dyabs, wl3), P._lowest_bit(h) * gq)
            P.check_product('dx GEMM', dY, wl, precision)
            dwl_abs += torch.einsum('i,ko->iok', x[c].abs(), dyabs)
        P.check_16bit('x rows of dW_L, application %d' % t, x, precision, normalise=True)
        P.check_sum('dW_L, application %d' % t, dwl_abs, P._lowest_bit(x) * P._lowest_bit(h) * gq)
        P.check_sum('db_L, application %d' % t, x[src].abs().t() @ G.abs(), P._lowest_bit(x) * gq)
    xs_scale = [torch.tensor([P._pow2_ge(float(v)) for v in x.abs().max(1).values]) for x in p.x]
    ghat = torch.cat([g[dst] * s[src].unsqueeze(1) for g, s in zip(p.grad_out, xs_scale)], 1)
    P.check_16bit('Ghat (MLP pass)', ghat, precision, normalise=True)
    dh, dh_abs = torch.zeros_like(h), torch.zeros_like(h)
    for x, g in zip(p.x, p.grad_out):
        Pm = (x[src].unsqueeze(2) * g[dst].unsqueeze(1)).reshape(-1, cin * cout)
        dh += Pm @ wl
        dh_abs += Pm.abs() @ wl.abs()
    P.check_sum('dh (k_dh)', dh_abs, min(P._lowest_bit(x) for x in p.x) * gq * P._lowest_bit(wl))
    P.check_product('k_dh Ghat . Y^T', ghat, torch.cat(p.x), precision)
    dz = dh * _grad(h)
    P.check_16bit('dz %d' % (len(ws) - 1), dz, precision, normalise=True)
    for l in range(len(ws) - 1, 0, -1):
        a = hs[l - 1]
        if l == 1:
            hi, lo = P._split(a, 'bf16' if precision == 'bf16' else 'f16')
            a_abs = hi.abs() + lo.abs() + 1
        else:
            a_abs = a.abs()
        qz = P._lowest_bit(dz)
        P.check_sum('dW_%d' % l, dz.abs().t() @ a_abs, qz * P._lowest_bit(a))
        P.check_sum('db_%d' % l, dz.abs().sum(0, keepdim=True), qz)
        P.check_product('dW_%d GEMM' % l, dz, a, precision)
        w = ws[l - 1]
        P.check_sum('d input of layer %d' % l, dz.abs() @ w.abs(), qz * P._lowest_bit(w))
        if l > 1:
            P.check_product('dz_%d GEMM' % (l - 1), dz, w, precision)
            dz = (dz @ w) * _grad(a)
            P.check_16bit('dz %d' % (l - 1), dz, precision, normalise=True)
