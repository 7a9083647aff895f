"""Exact integer probes of the NNConv paths.

A probe is an NNConv problem (graph, edge network, node features, optionally output gradients) whose every value is an
integer and whose magnitudes stay inside a budget: every value a kernel stores in a 16-bit buffer is exactly
representable there, and every fp32 sum stays within 2^22 quanta (the sum of the absolute values of its terms), so no
kernel rounds anywhere and every summation order gives the same bits.  With ``aggr='add'`` the library must then equal
the fp64 reference bit for bit, at every node and every gradient row: one lost, doubled or misrouted edge moves a node by
a whole message, and streamed, cached, fused and chained runs agree bitwise.

How a probe is built (``make_probe``):

* ``edge_attr`` is a small integer code hashed from ``(src, dst, column)``, so that messages differ from edge to edge
  (a misrouted edge changes two nodes, not zero).  With ``wide_ea`` every column of an edge also carries one common
  offset ``256 * b_e`` (b_e in 1..16): the values then need up to 13 significant bits, so the 16-bit hi/lo split of the
  tensor-core first layer has non-zero ``lo`` halves, and every first-layer unit reads two columns with weights +1 and
  -1, so the offset cancels exactly and the unit's value is a small integer again.
* every Linear of the edge network is sparse with entries in {-1, 0, +1}: a hidden unit is
  ``relu(h_a - h_b + bias)`` with a small integer bias, so activations stay small integers at any depth;
  the last Linear ``W_L`` has at most one input channel per (output channel, hidden unit) column, so every per-source
  matrix ``Y_src`` entry is +-1 times one entry of ``x_src`` (representable whenever ``x`` is).
* output channel 0 of every message is ``x_src[0] >= 1`` (the last bias ``b_L`` carries it, ``W_L`` has no row for it),
  so that no message is zero: deleting or duplicating an edge always changes its destination.
* ``x``, ``root``, ``bias`` and the output gradients are small integers.

``assert_exact(probe)`` proves, in fp64 on the CPU, that a probe meets the budget for its precision, and names the
buffer that does not.  The forward is checked over the distinct edge-attribute rows and the per-edge bounds derived from
them (so it runs at the 241^2 mesh); the backward quantities are computed edge by edge (small graphs only).
"""
import math

import numpy as np
import torch

SUM_QUANTA = 1 << 22                       # fp32 sums: sum |terms| <= 2^22 quanta
PAIR_OPERAND_BITS = 11                     # f16x2: one operand of every product has no lo half


# ---- integer hashing of edges (identical on every device) -------------------------------------------------------------
def _mix(v):
    v = v & 0xFFFFFFFF
    v = (v ^ (v >> 16)) * 0x45D9F3B & 0xFFFFFFFF
    v = (v ^ (v >> 16)) * 0x45D9F3B & 0xFFFFFFFF
    return v ^ (v >> 16)


def edge_hash(src, dst, salt):
    return _mix(_mix(src * 0x9E3779B1 + salt) + dst * 0x85EBCA77)


# ---- test graphs ------------------------------------------------------------------------------------------------------
def degree_graph(degrees, n_nodes, seed):
    """Source i has degrees[i] out-edges to random targets; edges in random order."""
    gen = torch.Generator().manual_seed(seed)
    src = torch.cat([torch.full((d,), i, dtype=torch.int64) for i, d in enumerate(degrees)])
    dst = torch.randint(0, n_nodes, (src.numel(),), generator=gen)
    perm = torch.randperm(src.numel(), generator=gen)
    return torch.stack([src[perm], dst[perm]])


# out-degrees whose last 128-edge tile holds every box height (16 * ceil(rows / 16)), plus one- and two-tile units
PARTIAL_TILE_DEGREES = [1, 15, 16, 17, 31, 33, 48, 50, 64, 65, 80, 90, 97, 100, 113, 120, 127, 128, 129, 200, 255, 256,
                        257, 300, 383, 384, 385, 511]


def mixed_graph(n_nodes=300, n_edges=5000, hub=700, seed=5):
    """Unsorted, directed: a hub source with ``hub`` out-edges, ten copies of one edge, 40 self-loops, targets 0..9
    without in-edges, and nodes n-10..n-1 isolated."""
    gen = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n_nodes - 20, (n_edges,), generator=gen)
    dst = torch.randint(10, n_nodes - 10, (n_edges,), generator=gen)
    src[:hub] = 7
    src[1000:1010] = src[1000]
    dst[1000:1010] = dst[1000]
    dst[2000:2040] = src[2000:2040].clamp(min=10)            # self-loops
    src[2000:2040] = dst[2000:2040]
    return torch.stack([src, dst])


def asymmetric_graph(n_nodes=200, n_edges=3000, seed=7):
    """A directed graph in which no edge has its reverse, with a hub source (node 3, ~390 out-edges) and a hub target
    (node 150, ~450 in-edges; the hub source under flow target_to_source): swapping src and dst gives a different
    graph, so a mix-up of the two ends cannot pass."""
    gen = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n_nodes, (n_edges,), generator=gen)
    dst = torch.randint(0, n_nodes, (n_edges,), generator=gen)
    src[:400] = 3
    dst[400:1000] = 150
    keep = src < dst                                        # an edge u -> v only for u < v: no reverse edges
    return torch.stack([src[keep], dst[keep]])


POW2_DEGREES = (1, 2, 4, 8, 16, 32, 64)
POW2_WEIGHTS = (.08, .10, .14, .20, .22, .18, .08)         # mean in-degree ~17, as in mixed_graph


def _pow2_choice(rng, size, max_in):
    """``size`` in-degrees drawn from POW2_DEGREES up to ``max_in`` (one number for size None)."""
    k = sum(d <= max_in for d in POW2_DEGREES)
    w = np.array(POW2_WEIGHTS[:k])
    return rng.choice(POW2_DEGREES[:k], size, p=w / w.sum())


def _pow2_layout(indeg, srcs_of_slots, rng):
    """One dst slot per in-edge of ``indeg`` (shuffled), paired with the sources ``srcs_of_slots(E)`` returns."""
    dst = np.repeat(np.arange(indeg.size), indeg)
    rng.shuffle(dst)
    return srcs_of_slots(dst), dst


def pow2_indegree_graph(n_nodes=300, hub=700, hub_in=256, seed=5, flow='source_to_target', max_in=64):
    """Every in-degree 0 or a power of two, so that aggr='mean' scales by exact 1/deg.  Unsorted, directed: a hub
    source (node 7, ``hub`` out-edges), a hub target (node n/2, ``hub_in`` in-edges), ten copies of one edge, 40
    self-loops, targets 0..9 without in-edges, and nodes n-10..n-1 isolated; the sources are random, so a node's
    out-degree differs from its in-degree at most nodes.  Built in (src, dst) terms; under ``flow='target_to_source'``
    the rows are stored swapped, so that the library reads the same (src, dst) pairs.  The other targets' in-degrees
    are powers of two up to ``max_in``."""
    rng = np.random.RandomState(seed)
    indeg = np.zeros(n_nodes, dtype=np.int64)
    targets = np.arange(10, n_nodes - 10)
    indeg[targets] = _pow2_choice(rng, targets.size, max_in)
    hub_t, dup_t, dup_s = n_nodes // 2, n_nodes // 3, 20
    indeg[hub_t], indeg[dup_t] = hub_in, 16
    indeg[dup_t] -= 10                                      # ten of its slots are the copies, laid out below
    src, dst = _pow2_layout(indeg, lambda d: rng.randint(0, n_nodes - 20, d.size), rng)
    src[:hub] = 7
    loops = np.arange(hub, hub + 40)
    src[loops] = dst[loops]                                 # self-loops
    src = np.concatenate([src, np.full(10, dup_s)])
    dst = np.concatenate([dst, np.full(10, dup_t)])
    perm = rng.permutation(src.size)
    src, dst = torch.from_numpy(src[perm]), torch.from_numpy(dst[perm])
    return torch.stack([dst, src] if flow == 'target_to_source' else [src, dst])


def pow2_degree_graph(out_degrees, n_nodes, seed, max_in=64):
    """Source i has out_degrees[i] out-edges; every target's in-degree is a power of two up to ``max_in`` (the
    remainder in its binary digits), edges in random order."""
    rng = np.random.RandomState(seed)
    E = int(sum(out_degrees))
    indeg = np.zeros(n_nodes, dtype=np.int64)
    left, order = E, rng.permutation(n_nodes)
    for n in order:
        if left == 0:
            break
        d = int(_pow2_choice(rng, None, max_in))
        d = d if d <= left else 1 << (left.bit_length() - 1)
        indeg[n], left = d, left - d
    assert left == 0, 'too few nodes for %d edges' % E

    def sources(d):
        s = np.repeat(np.arange(len(out_degrees)), out_degrees)
        rng.shuffle(s)
        return s
    src, dst = _pow2_layout(indeg, sources, rng)
    return torch.stack([torch.from_numpy(src), torch.from_numpy(dst)])


def pow2_low_degree_graph(n_src, seed):
    """Formulation B's shape with power-of-two in-degrees: 2-4 out-edges per source, in-degrees in {1, 2, 4, 8}."""
    rng = np.random.RandomState(seed)
    indeg = rng.choice([1, 2, 4, 8], n_src, p=[.25, .25, .4, .1])
    out = np.full(n_src, 3)
    delta = int(indeg.sum()) - 3 * n_src
    out[rng.permutation(n_src)[:abs(delta)]] += 1 if delta > 0 else -1

    def sources(d):
        s = np.repeat(np.arange(n_src), out)
        rng.shuffle(s)
        return s
    src, dst = _pow2_layout(indeg, sources, rng)
    return torch.stack([torch.from_numpy(src), torch.from_numpy(dst)])


def block_diagonal(graphs_and_sizes):
    """Disjoint union of (edge_index, n_nodes) pairs, node ids offset: a batch of graphs."""
    eis, off = [], 0
    for ei, n in graphs_and_sizes:
        eis.append(ei + off)
        off += n
    return torch.cat(eis, 1), off


# ---- the probe --------------------------------------------------------------------------------------------------------
class Probe(object):
    """x: list of T fp64 [N, cin] inputs (one per application), grad_out: list of T fp64 [N, cout] or None; ea: fp32
    [E, k_in] (integer valued, exact); ws, bs: fp64 edge-network parameters; root, bias: fp64 or None."""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    @property
    def T(self):
        return len(self.x)

    def src_dst(self):
        """(src, dst) rows of the edge index as the library reads them under this probe's flow."""
        ei = self.ei
        return (ei[1], ei[0]) if self.flow == 'target_to_source' else (ei[0], ei[1])

    def conv(self, cls, precision, aggr, device, **kw):
        from tests.helpers import make_conv
        conv = make_conv(cls, [w.float() for w in self.ws], [b.float() for b in self.bs],
                         None if self.root is None else self.root.float(),
                         None if self.bias is None else self.bias.float(), aggr, self.cin, self.cout, precision, device)
        conv.flow = self.flow
        for k, v in kw.items():
            setattr(conv, k, v)
        return conv


WIDE = 2048        # x = b + WIDE * a: 12 significant bits, so an f16x2 pair has a non-zero lo half


def make_probe(ei, n_nodes, layers, cin, cout, *, seed=0, T=1, grad=False, wide_ea=False, wide_x=False, wide_g=False,
               flow='source_to_target', y_density=1 / 16., g_density=1 / 8., g_rows=1.0, root_bias=True, g_in=None):
    """An exact probe on the graph ``ei`` (any device; the edge attributes are made on its device) for an edge network
    of widths ``layers`` (``layers[-1] == cin * cout``), with T inputs and, with ``grad``, T output gradients.
    ``wide_x`` / ``wide_g``: a quarter of the entries of x (channels >= 1) / of the non-zero output gradients get
    +-2048 added, so that they need 12 significant bits: the f16x2 pairs of Xc, Y, x, G, Ghat, dY and dz then have
    non-zero lo halves (one operand of every product keeps at most 11 bits, so lo * lo stays zero).  ``g_rows``: the
    fraction of nodes whose output-gradient rows may be non-zero; ``g_in``: if given, the in-degrees (under ``flow``)
    of the nodes whose output-gradient rows may be non-zero (aggr='mean': a narrow range of 1/deg keeps the 16-bit
    gradient buffers exact)."""
    assert layers[-1] == cin * cout
    rng = np.random.RandomState(seed)
    k_in = layers[0]
    src, dst = (ei[1], ei[0]) if flow == 'target_to_source' else (ei[0], ei[1])
    cols = [((edge_hash(src, dst, 101 + j) >> 7) % 4) for j in range(k_in)]
    ea = torch.stack(cols, 1).to(torch.float32)
    if wide_ea:
        ea = ea + (256 * (1 + (edge_hash(src, dst, 977) >> 9) % 16)).to(torch.float32).unsqueeze(1)
    n_lin = len(layers) - 1
    ws, bs = [], []
    for l in range(n_lin - 1):                                       # hidden layers: relu(h_a - h_b + bias)
        fan_in, fan_out = layers[l], layers[l + 1]
        w = np.zeros((fan_out, fan_in))
        a = rng.randint(0, fan_in, fan_out)
        b = (a + 1 + rng.randint(0, max(fan_in - 1, 1), fan_out)) % fan_in
        w[np.arange(fan_out), a] = 1
        if fan_in > 1:
            w[np.arange(fan_out), b] = -1
        ws.append(torch.from_numpy(w))
        bs.append(torch.from_numpy(rng.randint(-1, 3, fan_out).astype(np.float64)))
    K = layers[-2]
    wl = np.zeros((cin * cout, K))                                   # row i * cout + o
    for o in range(1, cout):
        pick = rng.rand(K) < y_density
        ks = np.nonzero(pick)[0]
        wl[rng.randint(0, cin, ks.size) * cout + o, ks] = rng.choice([-1, 1], ks.size)
    bl = np.zeros((cin, cout))
    bl[0, 0] = 1                                                     # message channel 0 = x_src[0] >= 1
    m = rng.rand(cin, cout - 1) < 0.1
    bl[:, 1:][m] = rng.choice([-1, 1], int(m.sum()))
    ws.append(torch.from_numpy(wl))
    bs.append(torch.from_numpy(bl.reshape(-1)))
    xs = []
    for _ in range(T):
        x = rng.randint(-3, 4, (n_nodes, cin)).astype(np.float64)
        x[:, 0] = rng.randint(1, 4, n_nodes)
        if wide_x:
            x[:, 1:] += WIDE * rng.choice([-1, 0, 0, 0, 0, 0, 0, 1], (n_nodes, cin - 1))
        xs.append(torch.from_numpy(x))
    root = bias = None
    if root_bias:
        root = torch.from_numpy(rng.choice([-1, 0, 0, 0, 1], (cin, cout)).astype(np.float64))
        root[:, 0] = 0                  # channel 0 = bias + the messages x_src[0]: a tight aggr='mean' bound there
        bias = torch.from_numpy(rng.randint(-2, 3, cout).astype(np.float64))
    gouts = None
    if grad:
        gouts = []
        for _ in range(T):
            g = rng.choice([-1, 1], (n_nodes, cout)) * (rng.rand(n_nodes, cout) < g_density)
            if g_rows < 1:
                g = g * (rng.rand(n_nodes, 1) < g_rows)
            if wide_g:
                g = g + WIDE * (g != 0) * rng.choice([-1, 0, 0, 0, 0, 0, 0, 1], (n_nodes, cout))
            if g_in is not None:
                deg = torch.bincount(dst.cpu(), minlength=n_nodes).numpy()
                g = g * np.isin(deg, g_in)[:, None]
            gouts.append(torch.from_numpy(g.astype(np.float64)))
    return Probe(ei=ei, n_nodes=n_nodes, flow=flow, layers=list(layers), cin=cin, cout=cout, ea=ea, ws=ws, bs=bs,
                 root=root, bias=bias, x=xs, grad_out=gouts, wide_ea=wide_ea)


# ---- the exactness proof ----------------------------------------------------------------------------------------------
class NotExact(AssertionError):
    pass


def _lowest_bit(t):
    """Smallest power of two dividing every non-zero entry (fp64), 1.0 for an all-zero tensor."""
    t = t[t != 0].abs()
    if t.numel() == 0:
        return 1.0
    mant, ex = torch.frexp(t)
    mi = (mant * 2.0 ** 53).to(torch.int64)
    low = mi & -mi
    return float(torch.min(torch.ldexp(low.double(), ex - 53)))


def significant_bits(t):
    """Largest number of significant bits of an entry (fp64 tensor; 0 for an all-zero tensor)."""
    t = t[t != 0].abs()
    if t.numel() == 0:
        return 0
    mant, _ = torch.frexp(t)
    mi = (mant * 2.0 ** 53).to(torch.int64)
    low = (mi & -mi).double()
    return int(53 - torch.log2(low).min().item())


def _pow2_ge(m):
    return 1.0 if m == 0 else 2.0 ** math.ceil(math.log2(m))


def roundtrip(v, precision):
    """v (fp64) through the 16-bit operand of ``precision``: one value, or an fp16 (hi, lo) pair at f16x2."""
    if precision == 'bf16':
        return v.to(torch.bfloat16).double()
    hi = v.to(torch.float16).double()
    if precision == 'f16x2':
        return hi + (v - hi).to(torch.float16).double()
    return hi


FP16_MIN_NORMAL = 2.0 ** -14


def check_16bit(name, v, precision, normalise=False, fp16_range=True, normal=False):
    """Every entry of ``v`` is stored unchanged by a 16-bit buffer (after the kernels' power-of-two normalisation by
    the largest magnitude, if ``normalise``), and inside the fp16 range where a raw fp16 value is stored.  ``normal``:
    no fp16 value (hi or lo half of an f16x2 pair) is subnormal -- the probes do not rely on every 16-bit writer and
    every MMA keeping fp16 subnormals."""
    if precision == 'fp32':
        return
    v = v.double()
    if normalise:
        v = v / _pow2_ge(float(v.abs().max()) if v.numel() else 0.0)
    elif fp16_range and precision != 'bf16' and v.numel() and float(v.abs().max()) > 65504:
        raise NotExact('%s: |value| %g beyond the fp16 range' % (name, float(v.abs().max())))
    bad = roundtrip(v, precision) != v
    if bool(bad.any()):
        raise NotExact('%s: %d of %d values are not exact in %s (e.g. %r)'
                       % (name, int(bad.sum()), v.numel(), precision, float(v[bad][0])))
    if normal and precision != 'bf16':
        halves = v.to(torch.float16).double().flatten()
        small = (halves != 0) & (halves.abs() < FP16_MIN_NORMAL)
        if bool(small.any()):
            raise NotExact('%s: %d values are fp16 subnormals (e.g. %r)' % (name, int(small.sum()),
                                                                           float(halves[small][0])))


def check_sum(name, abs_sum, quantum):
    """A sum whose terms have absolute values adding up to ``abs_sum``, each a multiple of ``quantum`` (a number, or
    a tensor of quanta that broadcasts against ``abs_sum``: one per sum)."""
    if abs_sum.numel() == 0:
        return
    if torch.is_tensor(quantum):
        worst = float((abs_sum / quantum).max())
    else:
        worst = float(abs_sum.max()) / quantum
    if worst > SUM_QUANTA:
        raise NotExact('%s: a sum reaches %.4g quanta, more than 2^22' % (name, worst))


def check_product(name, a, b, precision):
    """f16x2 drops lo(a) * lo(b): exact only when one operand of the product has no lo half."""
    if precision != 'f16x2':
        return
    ba, bb = significant_bits(a.double()), significant_bits(b.double())
    if min(ba, bb) > PAIR_OPERAND_BITS:
        raise NotExact('%s: both operands need more than %d bits (%d, %d): lo*lo would be dropped'
                       % (name, PAIR_OPERAND_BITS, ba, bb))


def _distinct_rows(ea):
    """(distinct rows, index of each row's distinct row).  A probe's row is its codes (ea mod 256, 2 bits each) and one
    common offset (ea // 256): one int64 key per row while that fits, a row sort otherwise."""
    E, k_in = ea.shape
    if E == 0:
        return ea, torch.zeros(0, dtype=torch.int64)
    if 2 * k_in + 8 <= 62 and bool((ea.remainder(256) < 4).all()) and bool((ea // 256 == ea[:, :1] // 256).all()):
        key = (ea[:, 0] // 256).to(torch.int64) << (2 * k_in)
        for j in range(k_in):
            key += ea[:, j].remainder(256).to(torch.int64) << (2 * j)
        keys, inv = torch.unique(key, return_inverse=True)
        first = torch.full((keys.numel(),), E, dtype=torch.int64).scatter_reduce(
            0, inv, torch.arange(E), 'amin')
        return ea[first], inv
    return torch.unique(ea, dim=0, return_inverse=True)


def _hidden(ea, ws, bs):
    """All activations [h_0 = ea, h_1, ..., h_{L-1}] of the edge network without its last Linear, fp64."""
    hs = [ea.double()]
    for w, b in zip(ws[:-1], bs[:-1]):
        hs.append(torch.relu(hs[-1] @ w.t() + b))
    return hs


def _split(v, precision):
    """hi and lo halves of the first layer's split operands."""
    dt = torch.bfloat16 if precision == 'bf16' else torch.float16
    hi = v.to(dt).double()
    return hi, v - hi


def in_degree_scale(probe, aggr):
    """Per-node factor of aggr ('add': 1, 'mean': 1 / max(in-degree, 1)) under the probe's flow, fp64 [N]."""
    if aggr == 'add':
        return torch.ones(probe.n_nodes, dtype=torch.float64)
    deg = torch.bincount(probe.src_dst()[1].cpu(), minlength=probe.n_nodes)
    return 1.0 / deg.clamp(min=1).double()


def assert_exact(probe, precision, kmat=None, aggr='add'):
    """Raise NotExact (naming the buffer) unless every kernel path computes ``probe`` without rounding at
    ``precision`` ('f16', 'bf16', 'f16x2' or 'fp32') and aggregation ``aggr`` ('add' or 'mean').  ``kmat``: also
    prove formulation B (per-edge kernel matrices; default: when the graph is small enough for the library to build
    them).  Returns the forward bounds used by the tests: a dict with the per-edge message bound ``msg`` [E] and the
    largest node sum ``node_sum``.

    aggr='mean' multiplies every message into node n by inv_deg[n] = 1 / deg(n) (and the backward every G and Ghat
    row of an edge into n): exact only when every in-degree is a power of two, and then a node's sum has quantum
    q * inv_deg[n].  Every fp16 value of a normalised buffer must also be normal (see ``check_16bit``)."""
    p = probe
    ws, bs = p.ws, p.bs
    ea = p.ea.double().cpu()
    src, dst = (t.cpu() for t in p.src_dst())
    E, N = ea.size(0), p.n_nodes
    if aggr not in ('add', 'mean'):
        raise ValueError(aggr)
    if aggr == 'mean':
        deg = torch.bincount(dst, minlength=N)
        odd = torch.nonzero((deg & (deg - 1)) != 0).flatten()
        if odd.numel():
            raise NotExact('in-degree: node %d has %d in-edges, not a power of two, so 1/deg is inexact (aggr=mean)'
                           % (int(odd[0]), int(deg[odd[0]])))
    inv_deg = in_degree_scale(p, aggr)
    n_lin = len(ws)
    single = n_lin == 1
    if kmat is None:
        kmat = E * p.cin * p.cout <= 1 << 30 and E > 0
    for l, (w, b) in enumerate(zip(ws, bs)):
        check_16bit('weight %d' % l, w, precision)
        check_16bit('bias %d' % l, b, precision)
    if p.root is not None:
        check_16bit('root', p.root, 'fp32')
    # the forward is a function of the distinct edge-attribute rows: prove it there
    uniq, inv = _distinct_rows(ea)
    hs = _hidden(uniq, ws, bs)
    if single:
        check_16bit('h (identity first layer: edge_attr)', uniq, precision)
    else:
        w1, b1 = ws[0], bs[0]
        if p.layers[0] <= 20:                       # tensor-core first layer: A1 = [hi(ea) | lo(ea) | hi(ea) | 1 | 1]
            hi, lo = _split(uniq, 'bf16' if precision == 'bf16' else 'f16')
            if precision != 'fp32':
                check_16bit('A1 hi(edge_attr)', hi, precision)
                check_16bit('A1 lo(edge_attr)', lo, precision)
                if not bool((hi + lo == uniq).all()):
                    raise NotExact('A1: hi + lo != edge_attr')
            s1 = (hi.abs() + lo.abs()) @ w1.abs().t() + b1.abs()
        else:                                       # CUDA-core first layer, fp32
            s1 = uniq.abs() @ w1.abs().t() + b1.abs()
        check_sum('first layer', s1, _lowest_bit(uniq) * _lowest_bit(w1))
        for l in range(1, n_lin):
            check_16bit('hidden activation %d' % l, hs[l], precision)
            if l >= 2:
                check_sum('hidden layer %d' % l, hs[l - 1].abs() @ ws[l - 1].abs().t() + bs[l - 1].abs(), 1.0)
                check_product('hidden layer %d' % l, hs[l - 1], ws[l - 1], precision)
    h = hs[-1]
    wl, bl = ws[-1], bs[-1]
    cin, cout = p.cin, p.cout
    wl3 = wl.view(cin, cout, -1)                                   # [i, o, k]
    if int((wl3 != 0).sum(0).max()) > 1:
        raise NotExact('W_L: a (channel, hidden unit) column reads more than one input channel')
    xq = min(_lowest_bit(x) for x in p.x)
    xmax = torch.stack([x.abs().max(1).values for x in p.x]).max(0).values         # per node
    for t, x in enumerate(p.x):
        check_16bit('Xc (x / per-source scale), input %d' % t, x / torch.tensor(
            [_pow2_ge(float(v)) for v in x.abs().max(1).values]).unsqueeze(1), precision)
        check_16bit('Y (one entry of x per column of W_L), input %d' % t, x, precision, normalise=True)
    check_product('contraction h . Y', h, torch.cat(p.x), precision)
    check_product('Y GEMM', torch.cat(p.x), wl, precision)
    wabs = wl3.abs().sum(0)                                        # [o, k]
    quantum = _lowest_bit(h) * _lowest_bit(wl) * xq
    c_abs = bl.abs().view(cin, cout)                               # |x| . |B3| <= xmax * colsum
    per_code = (h.abs() @ wabs.t()) + c_abs.sum(0)                 # [U, cout]: message bound / max|x_src|
    msg = per_code.max(1).values[inv] * xmax[src] if E else torch.zeros(0, dtype=torch.float64)
    check_sum('message (contraction + x . b_L)', msg, quantum)
    init = torch.zeros(N, dtype=torch.float64)
    if p.root is not None:
        init = init + xmax * p.root.abs().sum(0).max()
    if p.bias is not None:
        init = init + p.bias.abs().max()
    node_sum = init.index_add(0, dst, msg * inv_deg[dst])
    # node n's terms are multiples of quantum * inv_deg[n] (root and bias: of quantum)
    check_sum('scatter into out[dst] (root, bias and every in-edge)', node_sum,
              quantum * inv_deg if aggr == 'mean' else quantum)
    if kmat and precision in ('f16', 'bf16'):
        for c0 in range(0, h.size(0), 4096):
            kc = h[c0:c0 + 4096] @ wl.t() + bl
            check_16bit('K_e (formulation B)', kc, precision)
            check_sum('K_e build', h[c0:c0 + 4096].abs() @ wl.abs().t() + bl.abs(), _lowest_bit(h))
    if p.grad_out is not None:
        _assert_exact_backward(p, precision, src, dst, inv, hs, quantum, aggr, inv_deg)
    return {'msg': msg, 'node_sum': node_sum}


def _assert_exact_backward(p, precision, src, dst, inv, hs_u, q_fwd, aggr, inv_deg):
    """The tensor-core backward's 16-bit buffers and fp32 sums, edge by edge (nn_conv / backward_tc.cu):
    G_e = g[dst_e] * s_e; dY_c = sum_{e in c} h_e (x) G_e; dx, dW_L, db_L, droot, dbias; the MLP pass's
    Ghat_e[t] = g_t[dst_e] * s_e * xs_t[src_e] with Y_t = Xc_t W_L, dh_e = sum_t Ghat_e[t] . Y_t[src_e],
    dz_{L-1} = dh * mask, dz_{l-1} = (dz_l W_l) * mask, dW_l = dz_l^T h_{l-1}, dW_1 against A1,
    d edge_attr = dz_1 W_1.  s_e = inv_deg[dst_e] (1 for add): a sum over one source's edges (dY, dx) has the
    quantum of that source's smallest s_e, a sum over one edge's row (dh, dz W) that of its s_e, and a sum over every
    edge (dW_L, db_L, dW_l, db_l) that of the smallest s_e."""
    ws, bs = p.ws, p.bs
    cin, cout = p.cin, p.cout
    mean = aggr == 'mean'
    # an edge whose target has a zero gradient row in every application adds exact zeros to every buffer and sum below
    active = torch.stack([(g[dst] != 0).any(1) for g in p.grad_out]).any(0)
    src, dst, inv = src[active], dst[active], inv[active]
    s_e = inv_deg[dst]                                             # [E]
    s_min = float(s_e.min()) if s_e.numel() else 1.0
    hs = [a[inv] for a in hs_u]                                   # per active edge
    h = hs[-1]
    wl = ws[-1]
    order = torch.argsort(src, stable=True)
    counts = torch.bincount(src, minlength=p.n_nodes)
    s_src = torch.ones(p.n_nodes, dtype=torch.float64).scatter_reduce(0, src, s_e, 'amin')   # per source
    E = h.size(0)
    gq = min(_lowest_bit(g) for g in p.grad_out)
    for t, (x, g) in enumerate(zip(p.x, p.grad_out)):
        G = g[dst] * s_e.unsqueeze(1)
        check_16bit('G (gathered output gradient), application %d' % t, G, precision, normalise=True, normal=mean)
        # dY_c = h_c^T G_c  per source (in groups of sources), and the sums that read it
        if not bool(active.any()):
            continue
        check_product('k_dy h . G', h, G, precision)
        wl3 = wl.view(cin, cout, -1).abs()                         # [i, o, k]
        dwl_abs = torch.zeros_like(wl3)
        cs_all = torch.nonzero(counts).flatten().tolist()
        starts = torch.cumsum(counts, 0) - counts
        for g0 in range(0, len(cs_all), 256):
            cs = cs_all[g0:g0 + 256]
            dY = torch.stack([h[order[int(starts[c]):int(starts[c] + counts[c])]].t() @
                              G[order[int(starts[c]):int(starts[c] + counts[c])]] for c in cs])    # [S, K, cout]
            dyabs = torch.stack([h[order[int(starts[c]):int(starts[c] + counts[c])]].abs().t() @
                                 G[order[int(starts[c]):int(starts[c] + counts[c])]].abs() for c in cs])
            q_dy = _lowest_bit(h) * gq * (s_src[torch.tensor(cs)].view(-1, 1, 1) if mean else 1.0)
            check_sum('dY (k_dy), application %d' % t, dyabs, q_dy)
            check_16bit('dY, application %d' % t, dY, precision, normalise=True, normal=mean)
            # dx_c[i] = sum_{k,o} dY_c[k,o] W_L[i*cout+o, k]
            check_sum('dx = dY : W_L, application %d' % t, torch.einsum('sko,iok->si', dyabs, wl3),
                      q_dy.view(-1, 1) if mean else q_dy)
            check_product('dx GEMM', dY, wl, precision)
            check_product('dW_L GEMM', x, dY, precision)
            dwl_abs += torch.einsum('si,sko->iok', x[torch.tensor(cs)].abs(), dyabs)
        check_16bit('x rows of dW_L, application %d' % t, x, precision, normalise=True, normal=mean)
        check_sum('dW_L = x (x) dY, application %d' % t, dwl_abs, _lowest_bit(x) * _lowest_bit(h) * gq * s_min)
        check_sum('db_L, application %d' % t, x[src].abs().t() @ G.abs(), _lowest_bit(x) * gq * s_min)
    # MLP pass, all applications together
    xs_scale = [torch.tensor([_pow2_ge(float(v)) for v in x.abs().max(1).values]) for x in p.x]
    ghat = torch.cat([g[dst] * (s_e * s[src]).unsqueeze(1) for g, s in zip(p.grad_out, xs_scale)], 1)
    check_16bit('Ghat (MLP pass)', ghat, precision, normalise=True, normal=mean)
    dh = torch.zeros_like(h)
    dh_abs = torch.zeros_like(h)
    for x, g in zip(p.x, p.grad_out):
        P = (x[src].unsqueeze(2) * (g[dst] * s_e.unsqueeze(1)).unsqueeze(1)).reshape(E, cin * cout)
        dh += P @ wl
        dh_abs += P.abs() @ wl.abs()
    row_q = s_e.unsqueeze(1) if mean else 1.0                      # every term of edge e's row carries s_e
    check_sum('dh = Ghat . Y^T (k_dh)', dh_abs, min(_lowest_bit(x) for x in p.x) * gq * _lowest_bit(wl) * row_q)
    check_product('k_dh Ghat . Y^T', ghat, torch.cat(p.x), precision)
    n_lin = len(ws)
    if n_lin == 1:
        return
    dz = dh * (h > 0)
    check_16bit('dz %d' % (n_lin - 1), dz, precision, normalise=True, normal=mean)
    for l in range(n_lin - 1, 0, -1):                              # dz is the gradient at layer l's pre-activation
        a = hs[l - 1]
        if l == 1 and p.layers[0] <= 20:
            hi, lo = _split(a, 'bf16' if precision == 'bf16' else 'f16')
            a_abs = hi.abs() + lo.abs() + 1
        else:
            a_abs = a.abs()
        qz = _lowest_bit(dz)
        check_sum('dW_%d = dz^T h (k_gemm_tn)' % l, dz.abs().t() @ a_abs, qz * _lowest_bit(a))
        check_sum('db_%d' % l, dz.abs().sum(0, keepdim=True), qz)
        check_product('dW_%d GEMM' % l, dz, a, precision)
        w = ws[l - 1]
        qz_row = _lowest_bit(dz / row_q) * row_q if mean else qz
        check_sum('d input of layer %d = dz W' % l, dz.abs() @ w.abs(), qz_row * _lowest_bit(w))
        if l > 1:
            check_product('dz_%d GEMM' % (l - 1), dz, w, precision)
            dz = (dz @ w) * (a > 0)
            check_16bit('dz %d' % (l - 1), dz, precision, normalise=True, normal=mean)


# ---- the probes of the GPU tests (tests/test_probe_exactness.py proves every one of them) ------------------------------
KERNELNN = [6, 1024, 1024, 64 * 64]          # KernelNN's edge network at width 64, ker_width 1024


def low_degree_graph(n_src, seed):
    """2-4 out-edges per source (the per-edge kernel matrices of formulation B), unsorted."""
    deg = (torch.arange(n_src) * 7919 + seed) % 3 + 2
    return degree_graph(deg.tolist(), n_src, seed)


def graph(name):
    """(edge_index, n_nodes) of a named test graph (CPU)."""
    if name == 'mixed':
        return mixed_graph(), 300
    if name == 'partial_tiles':
        return degree_graph(PARTIAL_TILE_DEGREES, 600, seed=9), 600
    if name == 'hub_batches':                    # a hub of 2,500 out-edges among ~380 sources
        gen = torch.Generator().manual_seed(17)
        src = torch.randint(0, 380, (6000,), generator=gen)
        dst = torch.randint(0, 400, (6000,), generator=gen)
        src[:2500] = 200
        return torch.stack([src, dst]), 400
    if name == 'asymmetric':
        return asymmetric_graph(), 200
    if name == 'batch':
        return block_diagonal([graph('mixed'), graph('asymmetric'), (degree_graph([3, 130, 1, 257], 50, seed=4), 50)])
    if name == 'low_degree_4096':
        return low_degree_graph(4096, 1), 4096
    if name == 'low_degree_256':
        return low_degree_graph(256, 2), 256
    # power-of-two in-degrees (aggr='mean'), every graph in the (src, dst) rows of flow source_to_target but the t2s
    # one; suffix '_in32': in-degrees up to 32 (hub target included), for the probes with 12-bit x or g
    if name.startswith('pow2_'):
        base, max_in = (name[:-5], 32) if name.endswith('_in32') else (name, 64)
        hub_in, sfx = (256, '') if max_in == 64 else (max_in, '_in32')
        if base == 'pow2_mixed':
            return pow2_indegree_graph(hub_in=hub_in, max_in=max_in), 300
        if base == 'pow2_t2s':                   # another graph of the same kind, rows stored (dst, src)
            return pow2_indegree_graph(hub_in=hub_in, seed=6, flow='target_to_source', max_in=max_in), 300
        if base == 'pow2_partial_tiles':
            return pow2_degree_graph(PARTIAL_TILE_DEGREES, 600, seed=9, max_in=max_in), 600
        if base == 'pow2_hub_batches':           # a hub of 2,500 out-edges among ~380 sources
            return pow2_indegree_graph(400, hub=2500, hub_in=hub_in, seed=17, max_in=max_in), 400
        if base == 'pow2_batch':                 # a union keeps every in-degree
            return block_diagonal([graph('pow2_mixed' + sfx), (graph('pow2_t2s' + sfx)[0].flip(0), 300),
                                   (pow2_degree_graph([3, 130, 1, 257], 50, seed=4, max_in=max_in), 50)])
        if base == 'pow2_low_degree_4096':
            return pow2_low_degree_graph(4096, 1), 4096
        if base == 'pow2_low_degree_256':
            return pow2_low_degree_graph(256, 2), 256
    if name == 'darcy241':
        from oracle import nnconv_oracle as O
        return torch.from_numpy(O.ball_connectivity(241, 0.05)), 241 * 241
    if name == 'darcy85':
        from oracle import nnconv_oracle as O
        return torch.from_numpy(O.ball_connectivity(85, 0.10)), 85 * 85
    raise KeyError(name)


# name: (graph, layers, cin, cout, make_probe options, precisions it is used at)
FORWARD = {
    'mixed': ('mixed', [6, 64, 128, 64 * 64], 64, 64, {}, ('f16', 'bf16', 'f16x2', 'fp32')),
    'mixed_wide_ea': ('mixed', [6, 64, 128, 64 * 64], 64, 64, {'wide_ea': True}, ('f16', 'bf16', 'f16x2')),
    'partial_tiles': ('partial_tiles', [6, 32, 128, 64 * 64], 64, 64, {}, ('f16', 'bf16', 'f16x2')),
    'hub_batches': ('hub_batches', [6, 64, 256, 64 * 64], 64, 64, {}, ('f16', 'bf16', 'f16x2')),
    'asymmetric_t2s': ('asymmetric', [6, 64, 128, 64 * 64], 64, 64, {'flow': 'target_to_source'},
                       ('f16', 'bf16', 'f16x2')),
    'batch': ('batch', [6, 64, 128, 64 * 64], 64, 64, {}, ('f16', 'bf16', 'f16x2')),
    'nc16': ('mixed', [6, 64, 128, 16 * 16], 16, 16, {}, ('f16', 'bf16', 'f16x2')),
    'nc32': ('mixed', [6, 64, 128, 32 * 32], 32, 32, {}, ('f16', 'bf16', 'f16x2')),
    'nc48': ('mixed', [6, 64, 128, 48 * 48], 48, 48, {}, ('f16', 'bf16', 'f16x2')),
    'out80': ('mixed', [6, 64, 128, 64 * 80], 64, 80, {}, ('f16', 'bf16')),
    'out96': ('mixed', [6, 64, 128, 32 * 96], 32, 96, {}, ('f16', 'bf16')),
    'out112': ('mixed', [6, 64, 128, 64 * 112], 64, 112, {}, ('f16', 'bf16')),
    'out128': ('mixed', [6, 64, 128, 32 * 128], 32, 128, {}, ('f16', 'bf16')),
    'kp1088': ('mixed', [6, 128, 1088, 64 * 64], 64, 64, {}, ('f16', 'bf16')),
    'kin24_2layer': ('mixed', [24, 128, 64 * 64], 64, 64, {}, ('f16', 'bf16')),
    'kin24_3layer': ('mixed', [24, 64, 256, 64 * 64], 64, 64, {}, ('f16', 'bf16')),
    'single_linear': ('mixed', [100, 64 * 64], 64, 64, {}, ('f16', 'bf16')),
    'fp32_out40': ('mixed', [6, 64, 128, 32 * 40], 32, 40, {}, ('fp32',)),
    'edge_v64_src': ('low_degree_4096', [4, 64, 64, 64 * 64], 64, 64, {}, ('f16', 'bf16')),
    'edge_v64': ('low_degree_256', [4, 64, 64, 64 * 64], 64, 64, {}, ('f16', 'bf16')),
    'edge_v32': ('low_degree_256', [4, 64, 64, 32 * 32], 32, 32, {}, ('f16', 'bf16')),
    'edge_scalar_src': ('low_degree_4096', [4, 64, 64, 16 * 64], 16, 64, {}, ('f16', 'bf16')),
    'edge_scalar': ('low_degree_256', [4, 64, 64, 48 * 48], 48, 48, {}, ('f16', 'bf16')),
    'darcy241': ('darcy241', KERNELNN, 64, 64, {}, ('f16', 'f16x2')),
}

BACKWARD = {
    'mixed': ('mixed', [6, 64, 128, 64 * 64], 64, 64, {'T': 2}, ('f16', 'bf16', 'f16x2', 'fp32')),
    'mixed_T1': ('mixed', [6, 64, 128, 64 * 64], 64, 64, {'T': 1}, ('f16',)),
    'mixed_T6': ('mixed', [6, 64, 128, 64 * 64], 64, 64, {'T': 6}, ('f16',)),
    'mixed_T7': ('mixed', [6, 64, 128, 64 * 64], 64, 64, {'T': 7}, ('f16',)),
    'mixed_T8': ('mixed', [6, 64, 128, 64 * 64], 64, 64, {'T': 8}, ('f16',)),
    'mixed_T13': ('mixed', [6, 64, 128, 64 * 64], 64, 64, {'T': 13}, ('f16',)),
    'asymmetric_t2s': ('asymmetric', [6, 64, 128, 64 * 64], 64, 64, {'T': 2, 'flow': 'target_to_source'},
                       ('f16', 'bf16', 'f16x2')),
    'cuda_core_out32': ('mixed', [6, 64, 128, 32 * 32], 32, 32, {'T': 2}, ('f16', 'fp32')),
    'cuda_core_in128': ('mixed', [6, 64, 128, 128 * 64], 128, 64, {'T': 2}, ('f16', 'fp32')),
    # config-2 size (E = 1,466,497): every source's tiles run, gradient rows non-zero at 1/64 of the targets
    'darcy85': ('darcy85', [6, 64, 256, 64 * 64], 64, 64, {'T': 2, 'g_rows': 1 / 64.}, ('f16', 'bf16', 'f16x2')),
}

# f16x2 probes whose x (forward) or x / g (backward) carry 12-bit values with non-zero lo halves; the others keep
# small integers, because their sums would leave the budget (hub targets, and ~423 in-edges per node at 241^2).
# Backward: make_probe options per wide operand (fewer gradient rows keep dW_L and dW_l within 2^22 quanta).
WIDE_F16X2 = {
    'forward': ('mixed', 'mixed_wide_ea', 'partial_tiles', 'hub_batches', 'nc16', 'nc32', 'nc48'),
    'backward': {'mixed': {'x': {'wide_x': True, 'g_rows': 0.25}, 'g': {'wide_g': True, 'g_rows': 0.125}},
                 'asymmetric_t2s': {'g': {'wide_g': True, 'g_rows': 0.25}}},
}


# aggr='mean' probes: every in-degree under the probe's flow is 0 or a power of two (graphs 'pow2_*'), so that 1/deg
# is exact and the library must equal the fp64 mean bit for bit, as for add.
MEAN_FORWARD = {
    'mixed': ('pow2_mixed', [6, 64, 128, 64 * 64], 64, 64, {}, ('f16', 'bf16', 'f16x2', 'fp32')),
    't2s': ('pow2_t2s', [6, 64, 128, 64 * 64], 64, 64, {'flow': 'target_to_source'}, ('f16', 'bf16', 'f16x2')),
    'batch': ('pow2_batch', [6, 64, 128, 64 * 64], 64, 64, {}, ('f16', 'bf16', 'f16x2')),
    'hub_batches': ('pow2_hub_batches', [6, 64, 256, 64 * 64], 64, 64, {}, ('f16', 'bf16', 'f16x2')),
    'partial_tiles': ('pow2_partial_tiles', [6, 32, 128, 64 * 64], 64, 64, {}, ('f16', 'bf16', 'f16x2')),
    'edge_v64_src': ('pow2_low_degree_4096', [4, 64, 64, 64 * 64], 64, 64, {}, ('f16', 'bf16')),
    'edge_v64': ('pow2_low_degree_256', [4, 64, 64, 64 * 64], 64, 64, {}, ('f16', 'bf16')),
    'edge_v32': ('pow2_low_degree_256', [4, 64, 64, 32 * 32], 32, 32, {}, ('f16', 'bf16')),
    'edge_scalar_src': ('pow2_low_degree_4096', [4, 64, 64, 16 * 64], 16, 64, {}, ('f16', 'bf16')),
    'edge_scalar': ('pow2_low_degree_256', [4, 64, 64, 48 * 48], 48, 48, {}, ('f16', 'bf16')),
}

MEAN_BACKWARD = {
    'mixed': ('pow2_mixed', [6, 64, 128, 64 * 64], 64, 64, {'T': 2}, ('f16', 'bf16', 'f16x2', 'fp32')),
    'mixed_T1': ('pow2_mixed', [6, 64, 128, 64 * 64], 64, 64, {'T': 1}, ('f16', 'bf16', 'f16x2')),
    'mixed_T7': ('pow2_mixed', [6, 64, 128, 64 * 64], 64, 64, {'T': 7}, ('f16', 'bf16')),
    'mixed_T13': ('pow2_mixed', [6, 64, 128, 64 * 64], 64, 64, {'T': 13}, ('f16', 'bf16', 'f16x2')),
    't2s': ('pow2_t2s', [6, 64, 128, 64 * 64], 64, 64, {'T': 2, 'flow': 'target_to_source'},
            ('f16', 'bf16', 'f16x2', 'fp32')),
    't2s_T1': ('pow2_t2s', [6, 64, 128, 64 * 64], 64, 64, {'T': 1, 'flow': 'target_to_source'}, ('f16', 'bf16', 'f16x2')),
    't2s_T7': ('pow2_t2s', [6, 64, 128, 64 * 64], 64, 64, {'T': 7, 'flow': 'target_to_source'}, ('f16', 'bf16')),
    't2s_T13': ('pow2_t2s', [6, 64, 128, 64 * 64], 64, 64, {'T': 13, 'flow': 'target_to_source'},
                ('f16', 'bf16', 'f16x2')),
    'batch': ('pow2_batch', [6, 64, 128, 64 * 64], 64, 64, {'T': 2}, ('f16', 'bf16')),
    'cuda_core_out32': ('pow2_mixed', [6, 64, 128, 32 * 32], 32, 32, {'T': 2}, ('f16', 'fp32')),
    'cuda_core_in128': ('pow2_mixed', [6, 64, 128, 128 * 64], 128, 64, {'T': 2}, ('f16', 'fp32')),
}

# Per-precision make_probe options of the mean probes.  A dY entry of the 700-edge hub source mixes terms scaled by
# 1/1 .. 1/256, and the 16-bit dY must hold it: at f16 the gradient rows are non-zero only at targets of in-degree 8 to
# 256, at half the density; at bf16 (8 bits) only at targets of in-degree 16.  At f16x2, x carries 12-bit values
# (lo halves) on the '_in32' graphs (in-degrees up to 32: a 256-edge hub target's message sum of 12-bit x leaves the
# 2^22 budget), and the gradient rows are non-zero at an eighth of the targets of in-degree 16, so that dz stays in the
# fp16 normal range.  12-bit output gradients do not fit at mean: the hub source's dY then spans more than the fp16
# normal range.
MEAN_OPTIONS = {
    'forward': {'f16x2': {'wide_x': True, 'graph': '_in32'}},
    'backward': {'f16': {'g_in': (8, 16, 32, 64, 256), 'g_density': 1 / 16.}, 'bf16': {'g_in': (16,)},
                 'f16x2': {'wide_x': True, 'g_rows': 0.125, 'g_in': (16,), 'graph': '_in32'}},
}
MEAN_PLAIN = ('edge_v64_src', 'edge_v64', 'edge_v32', 'edge_scalar_src', 'edge_scalar', 'cuda_core_out32',
              'cuda_core_in128')                 # formulation B and the CUDA-core shapes: the table's options only
MEAN_PLAIN_F16X2_FORWARD = ('batch', 'hub_batches', 'partial_tiles')    # small-integer x: 12-bit x leaves the budget


def wide_options(table, name, precision, wide='x'):
    """make_probe options of the f16x2 variant of a probe (``wide``: 'x' or 'g', the backward operand that carries the
    lo halves), else {}; for a probe of ``MEAN_FORWARD`` or ``MEAN_BACKWARD``, its options at ``precision``
    (``MEAN_OPTIONS``, where 'graph' is the suffix of the graph to use)."""
    if table is MEAN_FORWARD or table is MEAN_BACKWARD:
        if name in MEAN_PLAIN or (table is MEAN_FORWARD and name in MEAN_PLAIN_F16X2_FORWARD):
            return {}
        return dict(MEAN_OPTIONS['forward' if table is MEAN_FORWARD else 'backward'].get(precision, {}))
    if precision != 'f16x2':
        return {}
    if table is FORWARD:
        return {'wide_x': True} if name in WIDE_F16X2['forward'] else {}
    return WIDE_F16X2['backward'].get(name, {}).get(wide, {})


def probe(table, name, device='cpu', precision=None, wide='x'):
    """The probe ``name`` of ``FORWARD``, ``BACKWARD``, ``MEAN_FORWARD`` or ``MEAN_BACKWARD`` with its graph on
    ``device``; at precision 'f16x2' the variant with lo halves where the budget allows (``wide``: which backward
    operand carries them, 'x' or 'g')."""
    gname, layers, cin, cout, opts, _ = table[name]
    opts = dict(opts, **wide_options(table, name, precision, wide))
    ei, n = graph(gname + opts.pop('graph', ''))
    return make_probe(ei.to(device), n, layers, cin, cout, grad=table is BACKWARD or table is MEAN_BACKWARD, **opts)
