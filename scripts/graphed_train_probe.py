#!/usr/bin/env python
"""Eager training step against the same step replayed by GraphedTrainStep, on the reference's batch-size-1 training
workloads:

    python scripts/graphed_train_probe.py [--rounds N] [--warmup W] [--only cfg1|uai1_61|burgers1024]

* cfg1        -- KernelNN config 1: 16 x 16 grid, r = 0.25, width 32, ker_width 1024, depth 4;
* uai1_61     -- KernelNN on UAI1_full_resolution.py's training mesh: 61 x 61, radius_train = 0.1, width 64,
                 ker_width 1024, depth 6;
* burgers1024 -- the orthogonal MGKN of MGKN_orthogonal_burgers1d.py at its training size: s = 2^13 / 8 = 1024,
                 9 levels, width 64, ker_width 1024, depth 4.

Two copies of each model start from the same parameters.  The eager copy trains with torch.optim.Adam (default
options), the replayed one with Adam(capturable=True) through GraphedTrainStep, on the same sample.  The two step kinds
alternate in one run, each bracketed by a device synchronise and timed with the host clock.  Printed: the card and its
power limit, the median of each, and the largest relative parameter difference (max |a - b| / max |b| over the
parameter tensors) after all steps."""
import argparse
import os
import statistics
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)
from graph_pde_b200 import GraphedTrainStep, graphs  # noqa: E402
from graph_pde_b200.models import MGKN, KernelNN  # noqa: E402
from scripts.train_probe import _power_limit  # noqa: E402


class _Data(object):
    pass


def _kernelnn(s, r, width, ker_width, depth, dev):
    x6, ei, ea = graphs.darcy_sample(s, r, dev, seed=0)
    d = _Data()
    d.x, d.edge_index, d.edge_attr = x6, ei, ea
    y = torch.randn(s * s, 1, generator=torch.Generator().manual_seed(1)).to(dev)

    def factory():
        torch.manual_seed(0)
        return KernelNN(width, ker_width, depth, 6, in_width=6).to(dev)
    return factory, d, y, 'E=%d' % ei.size(1)


def _burgers(dev):
    s = 2 ** 13 // 8
    theta = torch.randn(s, generator=torch.Generator().manual_seed(0))
    X, ei, ea = graphs.multi_pole_grid1d(theta, s, is_periodic=True, device=dev)
    y = torch.randn(s, 1, generator=torch.Generator().manual_seed(1)).to(dev)

    def factory():
        torch.manual_seed(0)
        return MGKN(width=64, ker_width=1024, depth=4, ker_in=4, in_width=2, s=s).to(dev)
    return factory, (X, None, ei, ea), y, '%d levels, edge sets %s' % (len(X), [e.size(1) for e in ei])


WORKLOADS = {
    'cfg1': lambda dev: _kernelnn(16, 0.25, 32, 1024, 4, dev),
    'uai1_61': lambda dev: _kernelnn(61, 0.1, 64, 1024, 6, dev),
    'burgers1024': _burgers,
}


def _timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def run(name, dev, rounds, warmup):
    factory, data, y, desc = WORKLOADS[name](dev)
    model_e, model_g = factory(), factory()
    model_g.load_state_dict(model_e.state_dict())
    opt_e = torch.optim.Adam(model_e.parameters(), lr=1e-4)
    opt_g = torch.optim.Adam(model_g.parameters(), lr=1e-4, capturable=True)

    def loss_of(model):
        return lambda data, y: F.mse_loss(model(data).view(-1), y.view(-1))

    def eager():
        opt_e.zero_grad(set_to_none=True)
        loss = loss_of(model_e)(data, y)
        loss.backward()
        opt_e.step()

    t0 = time.perf_counter()
    step = GraphedTrainStep(loss_of(model_g), model_g, opt_g, data, y, warmup=warmup)
    t_build = time.perf_counter() - t0
    for _ in range(warmup):            # the eager copy takes as many steps as the replayed one
        eager()
        step.replay()
    times = {'eager': [], 'replay': []}
    for _ in range(rounds):
        times['eager'].append(_timed(eager))
        times['replay'].append(_timed(step.replay))
    diff, diff_name = max((float((a.detach() - b.detach()).abs().max() / b.detach().abs().max().clamp(min=1e-30)), n)
                          for (n, a), b in zip(model_g.named_parameters(), model_e.parameters()))
    me, mr = statistics.median(times['eager']), statistics.median(times['replay'])
    print('%s (%s): eager step median %.3f ms, replayed step median %.3f ms (%.2fx); construction %.2f s; '
          'max relative parameter difference after %d steps: %.2e (%s)'
          % (name, desc, me, mr, me / mr, t_build, warmup + rounds, diff, diff_name))
    print('  eager : %s' % ', '.join('%.3f' % v for v in times['eager']))
    print('  replay: %s' % ', '.join('%.3f' % v for v in times['replay']))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--only', choices=sorted(WORKLOADS), default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('graphed_train_probe.py measures on a CUDA device; none is available')
    dev = torch.device('cuda:0')
    print('device: %s, power limit: %s' % (torch.cuda.get_device_name(dev), _power_limit()))
    for name in ([args.only] if args.only else ['cfg1', 'uai1_61', 'burgers1024']):
        run(name, dev, args.rounds, args.warmup)


if __name__ == '__main__':
    main()
