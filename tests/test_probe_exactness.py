"""CPU: every exact probe the GPU tests use is exact at every precision it is used at -- each 16-bit buffer holds its
values unchanged and every fp32 sum stays within 2^22 quanta (tests/probes.py).  A probe that is not exact fails here,
naming the buffer, instead of later as a false kernel bug."""
import pytest
import torch

from tests import probes as P


@pytest.mark.parametrize('name,precision', [(n, p) for n, spec in P.FORWARD.items() for p in spec[-1]])
def test_forward_probe_is_exact(name, precision):
    P.assert_exact(P.probe(P.FORWARD, name, precision=precision), precision)


@pytest.mark.parametrize('name,precision,wide', [(n, p, w) for n, spec in P.BACKWARD.items() for p in spec[-1]
                                                 for w in (('x', 'g') if p == 'f16x2' else ('x',))])
def test_backward_probe_is_exact(name, precision, wide):
    P.assert_exact(P.probe(P.BACKWARD, name, precision=precision, wide=wide), precision)


@pytest.mark.parametrize('table,name', [(P.FORWARD, n) for n in P.WIDE_F16X2['forward']] +
                         [(P.BACKWARD, n) for n in P.WIDE_F16X2['backward']])
def test_f16x2_probes_have_lo_halves(table, name):
    """The f16x2 variants store values that need more than 11 bits: their pairs' lo halves are not all zero."""
    for wide in P.WIDE_F16X2['backward'][name] if table is P.BACKWARD else ('x',):
        p = P.probe(table, name, precision='f16x2', wide=wide)
        t = torch.cat(p.x if wide == 'x' else p.grad_out)
        assert P.significant_bits(t) > P.PAIR_OPERAND_BITS, (name, wide)
        assert bool((t - t.half().double() != 0).any()), (name, wide)


def test_probes_are_integer_and_messages_differ():
    """Integer values throughout, and edge attributes that differ between edges (a misrouted edge changes two nodes)."""
    p = P.probe(P.FORWARD, 'mixed')
    for t in [p.ea.double()] + p.ws + p.bs + p.x + [p.root, p.bias]:
        assert bool((t == t.round()).all())
    distinct = torch.unique(p.ea, dim=0).size(0)
    assert distinct > 0.5 * min(p.ea.size(0), 4 ** p.ea.size(1)), distinct


def test_a_probe_beyond_the_budget_is_refused():
    """The proof is not vacuous: a probe whose sums exceed 2^22 quanta, or whose values need more bits than bf16
    holds, is refused with the buffer's name."""
    p = P.probe(P.FORWARD, 'mixed')
    p.x = [x * 4099 for x in p.x]
    with pytest.raises(P.NotExact, match='Xc|scatter|message'):
        P.assert_exact(p, 'bf16')
    p = P.probe(P.FORWARD, 'mixed')
    p.x = [x * 2 ** 12 + 1 for x in p.x]
    with pytest.raises(P.NotExact, match='scatter'):
        P.assert_exact(p, 'f16x2')


# ---- aggr='mean': power-of-two in-degrees ------------------------------------------------------------------------------
@pytest.mark.parametrize('name,precision', [(n, p) for n, spec in P.MEAN_FORWARD.items() for p in spec[-1]])
def test_mean_forward_probe_is_exact(name, precision):
    P.assert_exact(P.probe(P.MEAN_FORWARD, name, precision=precision), precision, aggr='mean')


@pytest.mark.parametrize('name,precision', [(n, p) for n, spec in P.MEAN_BACKWARD.items() for p in spec[-1]])
def test_mean_backward_probe_is_exact(name, precision):
    P.assert_exact(P.probe(P.MEAN_BACKWARD, name, precision=precision), precision, aggr='mean')


def test_mean_f16x2_probes_have_lo_halves():
    for table, name in ((P.MEAN_FORWARD, 'mixed'), (P.MEAN_FORWARD, 't2s'), (P.MEAN_BACKWARD, 'mixed')):
        t = torch.cat(P.probe(table, name, precision='f16x2').x)
        assert P.significant_bits(t) > P.PAIR_OPERAND_BITS, name


@pytest.mark.parametrize('change', ['drop', 'add'])
def test_a_mean_probe_with_one_odd_in_degree_is_refused(change):
    """The mean proof is not vacuous: one node's in-degree moved from 4 to 3 (an in-edge dropped) or to 5 (one added)
    is refused by the degree clause, though every add budget still holds."""
    p = P.probe(P.MEAN_FORWARD, 'mixed', precision='f16')
    src, dst = p.src_dst()
    deg = torch.bincount(dst, minlength=p.n_nodes)
    node = int(torch.nonzero(deg == 4)[0])
    e = int(torch.nonzero(dst == node)[0])
    if change == 'drop':
        keep = torch.arange(dst.numel()) != e
        p.ei, p.ea = p.ei[:, keep], p.ea[keep]
    else:
        p.ei, p.ea = torch.cat([p.ei, p.ei[:, e:e + 1]], 1), torch.cat([p.ea, p.ea[e:e + 1]])
    P.assert_exact(p, 'f16')
    with pytest.raises(P.NotExact, match='in-degree: node %d has %d in-edges' % (node, 3 if change == 'drop' else 5)):
        P.assert_exact(p, 'f16', aggr='mean')


def _fp64_mean(p, edge_scale):
    """fp64 (out, dx) of the first application with each message and gradient row scaled by edge_scale [E]."""
    from oracle import nnconv_oracle as O
    src, dst = p.src_dst()
    k = O.dense_net(p.ea.double(), p.ws, p.bs).view(-1, p.cin, p.cout)
    msg = torch.bmm(p.x[0][src].unsqueeze(1), k).squeeze(1) * edge_scale.unsqueeze(1)
    out = torch.zeros(p.n_nodes, p.cout, dtype=torch.float64).index_add(0, dst, msg)
    g = p.grad_out[0][dst] * edge_scale.unsqueeze(1)
    dx = torch.zeros(p.n_nodes, p.cin, dtype=torch.float64).index_add(0, src, torch.bmm(k, g.unsqueeze(2)).squeeze(2))
    return out, dx


@pytest.mark.parametrize('table,name', [(P.MEAN_BACKWARD, n) for n in ('mixed', 't2s', 'batch')] +
                         [(P.MEAN_FORWARD, n) for n in ('hub_batches', 'partial_tiles', 'edge_v64_src', 'edge_v64')])
def test_a_degree_read_at_the_wrong_end_changes_most_nodes(table, name):
    """On the mean probes, the fp64 mean with 1/deg taken from the source end of each edge (its in-degree), or with a
    node's out-degree in place of its in-degree, differs from the true mean at most nodes with in-edges (out) and at
    most sources whose out-edges meet a gradient row (dx): a kernel that mixes up the ends cannot pass."""
    p = P.probe(table, name, precision='f16')
    if p.grad_out is None:
        p.grad_out = [torch.ones(p.n_nodes, p.cout, dtype=torch.float64)]
    src, dst = p.src_dst()
    indeg = torch.bincount(dst, minlength=p.n_nodes).clamp(min=1).double()
    outdeg = torch.bincount(src, minlength=p.n_nodes).clamp(min=1).double()
    out, dx = _fp64_mean(p, 1.0 / indeg[dst])
    has_in = torch.bincount(dst, minlength=p.n_nodes) > 0
    feeds = torch.zeros(p.n_nodes, dtype=torch.bool).index_fill_(0, src[(p.grad_out[0][dst] != 0).any(1)], True)
    for wrong in (1.0 / indeg[src], 1.0 / outdeg[dst]):
        out_w, dx_w = _fp64_mean(p, wrong)
        assert float(((out_w != out).any(1) & has_in).sum()) > 0.5 * float(has_in.sum())
        assert float(((dx_w != dx).any(1) & feeds).sum()) > 0.5 * float(feeds.sum())
