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
