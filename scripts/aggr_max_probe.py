"""aggr='mean' against aggr='max' on one card, alternating the two (three rounds by default) so that clock and
thermal drift fall on both alike:

* darcy241 f16 (bench.py's configuration: KernelNN width 64, ker_width 1024, T = 6): the forward step (edge features
  recomputed every step, as bench.py's main number) and the fused application kernel per application (CUDA events
  around every k_apply_tc launch, nnconv_profile_*);
* a KernelNN training step (forward + backward + Adam) at 85^2, r = 0.10, f16 and f16x2.

Prints one JSON object (and writes it to --out) with the card name and power limit read in the same run.

    python scripts/aggr_max_probe.py [--rounds 3] [--steps 5] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from graph_pde_b200 import _lib, graphs, nn_conv  # noqa: E402
from graph_pde_b200.models import KernelNN  # noqa: E402

PK_APPLY_FUSED = 5


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [v.strip() for v in q.split(',')]
        return name, limit
    except Exception as e:      # the numbers still mean something with the name from torch
        return torch.cuda.get_device_name(), 'unknown (%s)' % type(e).__name__


def timed(fn, steps, warmup):
    for i in range(warmup):
        fn(i)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(steps):
        fn(warmup + i)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


class D(object):
    pass


def forward_241(dev, steps):
    torch.manual_seed(0)
    model = KernelNN(64, 1024, 6, 6, in_width=6, precision='f16').to(dev).eval()
    ei = graphs.ball_connectivity(241, 0.05, dev, True)
    x, _, ea = graphs.darcy_sample(241, 0.05, dev, seed=0, edge_index=ei)
    L = _lib.lib()

    def step(i):
        model.conv1._h_cache.clear()          # a new sample every step: the edge features are recomputed
        with torch.no_grad():
            return model.conv_stack(model.fc1(x), ei, ea)

    def measure(aggr):
        model.conv1.aggr = aggr
        ms = timed(step, steps, 2)
        _lib.check(L.nnconv_profile_begin())
        step(0)
        ms_k = (ctypes.c_double * 8)()
        n_k = (ctypes.c_int64 * 8)()
        _lib.check(L.nnconv_profile_end(ms_k, n_k, 8))
        return dict(step_ms=ms, apply_ms=ms_k[PK_APPLY_FUSED] / max(int(n_k[PK_APPLY_FUSED]), 1),
                    apply_launches=int(n_k[PK_APPLY_FUSED]))
    return measure, lambda: model.conv1.invalidate()


def train_85(dev, precision, steps):
    torch.manual_seed(0)
    model = KernelNN(64, 1024, 6, 6, in_width=6, precision=precision).to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=1e-4)
    ei = graphs.ball_connectivity(85, 0.10, dev, True)
    x, _, ea = graphs.darcy_sample(85, 0.10, dev, seed=0, edge_index=ei)
    y = torch.randn(85 * 85, 1, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    d = D()
    d.x, d.edge_index, d.edge_attr = x, ei, ea

    def step(i):
        opt.zero_grad(set_to_none=True)
        loss = torch.norm(model(d).view(-1) - y.view(-1), 1)
        loss.backward()
        opt.step()

    def measure(aggr):
        model.conv1.aggr = aggr
        model.conv1.invalidate()
        return dict(step_ms=timed(step, steps, 2))
    return measure, lambda: model.conv1.invalidate()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    dev = torch.device('cuda', torch.cuda.current_device())
    _lib.check(_lib.lib().nnconv_init())
    name, limit = card()
    res = dict(card=name, power_limit=limit, rounds=args.rounds, steps=args.steps, cases={})
    cases = [('darcy241_f16_forward', lambda: forward_241(dev, args.steps)),
             ('darcy85_f16_train', lambda: train_85(dev, 'f16', args.steps)),
             ('darcy85_f16x2_train', lambda: train_85(dev, 'f16x2', args.steps))]
    for case, make in cases:
        measure, release = make()
        runs = {'mean': [], 'max': []}
        for _ in range(args.rounds):
            for aggr in ('mean', 'max'):
                runs[aggr].append(measure(aggr))
        release()
        torch.cuda.empty_cache()
        summary = {}
        for aggr, rs in runs.items():
            for k in rs[0]:
                vals = sorted(r[k] for r in rs)
                summary['%s_%s' % (aggr, k)] = dict(median=vals[len(vals) // 2], min=vals[0], max=vals[-1])
        summary['max_over_mean_step'] = summary['max_step_ms']['median'] / summary['mean_step_ms']['median']
        if 'max_apply_ms' in summary:
            summary['max_over_mean_apply'] = summary['max_apply_ms']['median'] / summary['mean_apply_ms']['median']
        res['cases'][case] = summary
    res['launches_note'] = 'stats launches per forward differ by one finalize launch per max application'
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
