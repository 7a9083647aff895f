#!/usr/bin/env python
"""What the hidden activation of the edge network costs on the GPU, against ReLU:

    python scripts/edge_activation_probe.py [--rounds N] [--skip-241] [--accuracy]

1. The edge-feature pass of KernelNN's edge network [6, 1024, 1024, 64 * 64] over the 85^2 Darcy graph (E = 1,466,497)
   at f16: the CUDA-event time of the whole pass and the torch.profiler time of its hidden-layer GEMM (the 1024 x 1024
   k_gemm_tc launches, every second GEMM of the pass: the first layer's and the hidden layer's alternate per chunk).
2. One KernelNN training step at 85^2 (f16, tensor-core backward, Adam), per activation.
3. One KernelNN forward at 241^2 (f16, T = 6, edge features recomputed as for a new sample) with Tanh and with ReLU.
Rounds alternate the activations, and the median is printed with the device and its power limit.  --accuracy prints,
instead, max|out - ref| / max|ref| of the forward and of every gradient against fp64 autograd (tests/act_oracle.py)
per activation and precision, on the 12,000-edge hub graph of tests/test_gpu_edge_activation.py (aggr mean, T = 2)."""
import argparse
import os
import statistics
import sys

import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)
from bench import WORKLOADS  # noqa: E402
from graph_pde_b200 import graphs, nn_conv  # noqa: E402
from graph_pde_b200.models import DenseNet, KernelNN  # noqa: E402
from scripts.train_probe import _power_limit, _timed  # noqa: E402

ACTS = [('relu', torch.nn.ReLU), ('leaky_relu', lambda: torch.nn.LeakyReLU(0.01)), ('elu', torch.nn.ELU),
        ('tanh', torch.nn.Tanh), ('sigmoid', torch.nn.Sigmoid), ('relu6', torch.nn.ReLU6),
        ('hardtanh', lambda: torch.nn.Hardtanh(-0.3, 0.7)), ('hardsigmoid', torch.nn.Hardsigmoid), ('selu', torch.nn.SELU),
        ('celu', lambda: torch.nn.CELU(0.5)), ('softsign', torch.nn.Softsign), ('logsigmoid', torch.nn.LogSigmoid)]


class _Data(object):
    pass


def _set_activation(model, factory):
    layers = model.conv1.nn.layers
    for i, layer in enumerate(layers):
        if not isinstance(layer, torch.nn.Linear):
            layers[i] = factory()
    model.conv1.invalidate()


def _edge_feature_pass(dev, rounds):
    cfg = WORKLOADS['darcy85']
    x6, ei, ea = graphs.darcy_sample(cfg['s'], cfg['r'], dev, seed=0)
    n = x6.size(0)
    res = {}
    convs = {}
    for name, factory in ACTS:
        torch.manual_seed(0)
        convs[name] = nn_conv.NNConv_old(64, 64, DenseNet([6, 1024, 1024, 64 * 64], factory), aggr='mean',
                                         precision='f16').to(dev)
    plan = nn_conv.get_plan(ei, n)

    def one(conv):
        conv._h_cache.clear()
        conv.edge_features(plan, conv._get_prepared('f16'), ea)

    for conv in convs.values():
        one(conv)
    torch.cuda.synchronize()
    times = {name: [] for name, _ in ACTS}
    for _ in range(rounds):
        for name, _ in ACTS:
            times[name].append(_timed(lambda: one(convs[name])))
    for name, _ in ACTS:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            one(convs[name])
            torch.cuda.synchronize()
        gemms = sorted((e for e in prof.events() if 'k_gemm_tc' in e.name), key=lambda e: e.time_range.start)
        hidden = [e.time_range.elapsed_us() for e in gemms[1::2]]         # [first layer, hidden layer] per chunk
        first = [e.time_range.elapsed_us() for e in gemms[0::2]]
        res[name] = (statistics.median(times[name]), sum(hidden) / 1e3, sum(first) / 1e3, len(hidden))
        convs[name]._h_cache.clear()
    print('85^2 edge-feature pass, f16, [6, 1024, 1024, 4096], E=%d (median of %d rounds):' % (ei.size(1), rounds))
    for name, (t, h, f, k) in res.items():
        print('  %-10s pass %8.2f ms (%+.1f %% vs relu)   hidden GEMM %8.2f ms in %d launches (%+.1f %%)   first layer '
              '%6.2f ms' % (name, t, 100 * (t / res['relu'][0] - 1), h, k, 100 * (h / res['relu'][1] - 1), f))
    del convs
    torch.cuda.empty_cache()


def _training_step(dev, rounds):
    cfg = WORKLOADS['darcy85']
    s, r, w, kw, T = cfg['s'], cfg['r'], cfg['width'], cfg['ker_width'], cfg['depth']
    torch.manual_seed(0)
    model = KernelNN(w, kw, T, 6, in_width=6, precision='f16').to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=1e-4)
    x6, ei, ea = graphs.darcy_sample(s, r, dev, seed=0)
    y = torch.randn(s * s, 1, device=dev)
    d = _Data()
    d.x, d.edge_index, d.edge_attr = x6, ei, ea

    def step():
        opt.zero_grad(set_to_none=True)
        loss = torch.norm(model(d).view(-1) - y.view(-1), 1)
        loss.backward()
        opt.step()

    times = {name: [] for name, _ in ACTS}
    for name, factory in ACTS:                                 # warm-up: every activation's kernels
        _set_activation(model, factory)
        step()
    torch.cuda.synchronize()
    for _ in range(rounds):
        for name, factory in ACTS:
            _set_activation(model, factory)
            times[name].append(_timed(step))
    base = statistics.median(times['relu'])
    print('85^2 KernelNN training step, f16, E=%d, T=%d (median of %d rounds):' % (ei.size(1), T, rounds))
    for name, _ in ACTS:
        t = statistics.median(times[name])
        print('  %-10s %8.2f ms (%+.1f %% vs relu)  all: %s' % (name, t, 100 * (t / base - 1),
                                                              ', '.join('%.1f' % v for v in times[name])))
    del model, opt
    torch.cuda.empty_cache()


def _forward_241(dev, rounds):
    cfg = WORKLOADS['darcy241']
    s, r, w, kw, T = cfg['s'], cfg['r'], cfg['width'], cfg['ker_width'], cfg['depth']
    torch.manual_seed(0)
    model = KernelNN(w, kw, T, 6, in_width=6, precision='f16').to(dev)
    x6, ei, ea = graphs.darcy_sample(s, r, dev, seed=0)
    d = _Data()
    d.x, d.edge_index, d.edge_attr = x6, ei, ea
    acts = [ACTS[0], ACTS[3]]

    def step():
        model.conv1.invalidate()                               # a new sample: its edge features are computed again
        with torch.no_grad():
            model(d)

    times = {name: [] for name, _ in acts}
    for name, factory in acts:
        _set_activation(model, factory)
        step()
    torch.cuda.synchronize()
    for _ in range(rounds):
        for name, factory in acts:
            _set_activation(model, factory)
            times[name].append(_timed(step))
    base = statistics.median(times['relu'])
    print('241^2 KernelNN forward, f16, E=%d, T=%d, edge features recomputed per step (median of %d rounds):'
          % (ei.size(1), T, rounds))
    for name, _ in acts:
        t = statistics.median(times[name])
        print('  %-10s %8.1f ms (%+.1f %% vs relu)  all: %s' % (name, t, 100 * (t / base - 1),
                                                              ', '.join('%.1f' % v for v in times[name])))


def _accuracy():
    from tests import test_gpu_edge_activation as G0
    from tests import test_gpu_edge_activation_more as G1
    from tests.helpers import rel_err
    nn_conv._EDGE_KERNELS = 'off'
    ei, n = G0._hub_graph()
    ea, xs, gs = G0._inputs(ei, n, T=2)
    print('max|err| / max|ref| against fp64 (forward; worst parameter / x gradient; edge_attr gradient), aggr mean, '
          'E=%d, T=2, [6, 128, 128, 64 * 64]:' % ei.size(1))
    for G, kind, p in [(G, kind, p) for G in (G0, G1) for kind, p in G.ACTS]:   # G1: first layer scaled by 4
        for precision in ('f16', 'bf16', 'f16x2', 'fp32'):
            conv = G._conv(kind, p, precision, 'mean')
            with torch.no_grad():
                fwd = rel_err(conv(xs[0].to('cuda'), ei.to('cuda'), ea.to('cuda')),
                              G._oracle_out(conv, kind, p, xs[0], ei, ea, 'mean'))
            conv.invalidate()
            got = G._library_grads(conv, ei, ea, xs, gs)
            ref = G._reference_grads(conv, kind, p, ei, ea, xs, gs)
            k = G._ea_index(conv)
            errs = [rel_err(a, b) for a, b in zip(got, ref)]
            print('  %-10s %-5s  forward %.2e   gradients %.2e   edge_attr %.2e'
                  % (kind, precision, fwd, max(e for i, e in enumerate(errs) if i != k), errs[k]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--skip-241', action='store_true')
    ap.add_argument('--accuracy', action='store_true')
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    print('device: %s, power limit: %s' % (torch.cuda.get_device_name(dev), _power_limit()))
    if args.accuracy:
        _accuracy()
        return
    _edge_feature_pass(dev, args.rounds)
    _training_step(dev, args.rounds)
    if not args.skip_241:
        _forward_241(dev, max(args.rounds // 2, 2))


if __name__ == '__main__':
    main()
