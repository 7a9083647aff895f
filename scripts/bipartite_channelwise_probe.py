"""Time the bipartite DiagNNConv and GaussianNNConv against the same maps run as square convs on the union graph
(DESIGN 4.10):

    python scripts/bipartite_channelwise_probe.py [--reps 5] [--precision f16] [--out result.json]

The graph is scripts/bipartite_probe.py's: sources on the 121 x 121 mesh of [0, 1]^2, targets on the 241 x 241 query
points, an edge from every source within r = 0.05 of a target.  Width C = 64 on both sides, aggr='mean'.  DiagNNConv's
edge network is DenseNet([6, 512, 1024, 64]) on (x_src, x_dst, a_src, a_dst); GaussianNNConv reads (|x_src - x_dst|,
1 + a_src, 1 + a_dst), so every amplitude 1 / sqrt(|p1 p2|) is finite, and its sigma comes from Linear(1, 64).  For each
conv and form: one forward under no_grad (DiagNNConv's d cached, as a trained GKN evaluates) and one training step
(forward + backward through x_src, x_dst, edge_attr and every parameter; d rebuilt each step).  The two forms alternate
within one process, so the spread between repetitions is measured beside the difference.  Prints one JSON line with the
card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bipartite_probe import ball_edges, mesh, timed  # noqa: E402


def power_limit():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                              stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        return 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--precision', default='f16')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bipartite_channelwise_probe: no CUDA device (timings are GPU-only)')
    from graph_pde_b200.gauss import GaussianNNConv
    from graph_pde_b200.nn_conv import DiagNNConv
    from tests.helpers import DenseNetLike
    dev = 'cuda'
    C = 64
    ps, pd = mesh(121).to(dev), mesh(241).to(dev)
    ns, nd = ps.size(0), pd.size(0)
    ei = ball_edges(ps, pd, 0.05)
    g = torch.Generator(device=dev).manual_seed(0)
    a_s, a_d = torch.rand(ns, 1, device=dev, generator=g), torch.rand(nd, 1, device=dev, generator=g)
    ea_diag = torch.cat([ps[ei[0]].float(), pd[ei[1]].float(), a_s[ei[0]], a_d[ei[1]]], 1)
    ea_gauss = torch.cat([(ps[ei[0]] - pd[ei[1]]).norm(dim=1, keepdim=True).float(), 1 + a_s[ei[0]], 1 + a_d[ei[1]]], 1)
    union = torch.stack([ei[0], ei[1] + ns])
    xs = torch.randn(ns, C, device=dev, generator=g)
    xd = torch.randn(nd, C, device=dev, generator=g)
    xu = torch.cat([xs, xd])
    gd = torch.randn(nd, C, device=dev, generator=g)
    torch.manual_seed(0)
    convs = {'diag': (DiagNNConv(C, C, DenseNetLike([6, 512, 1024, C]), aggr='mean', precision=args.precision).to(dev),
                      ea_diag),
             'gauss': (GaussianNNConv(C, C, torch.nn.Linear(1, C), aggr='mean').to(dev), ea_gauss)}
    res = {'card': torch.cuda.get_device_name(0), 'power_limit': power_limit(), 'n_src': ns, 'n_dst': nd,
           'edges': int(ei.size(1)), 'channels': C, 'aggr': 'mean', 'diag_precision': args.precision}
    for kind, (conv, ea) in convs.items():
        def fwd_bip():
            with torch.no_grad():
                return conv((xs, xd), ei, ea)

        def fwd_union():
            with torch.no_grad():
                return conv(xu, union, ea)[ns:]

        def step_bip():
            a, b, e = xs.clone().requires_grad_(), xd.clone().requires_grad_(), ea.clone().requires_grad_()
            (conv((a, b), ei, e) * gd).sum().backward()

        def step_union():
            x, e = xu.clone().requires_grad_(), ea.clone().requires_grad_()
            (conv(x, union, e)[ns:] * gd).sum().backward()

        ref = fwd_union()
        res[kind + '_rel_diff_bip_vs_union'] = float((fwd_bip() - ref).abs().max() / ref.abs().max())
        for name, fn in (('forward', (fwd_bip, fwd_union)), ('train_step', (step_bip, step_union))):
            for f in fn:
                f()                               # warm-up: plans, d, workspaces
            tb, tu = [], []
            for _ in range(args.reps):            # alternate the two forms
                tb += timed(fn[0], 1)
                tu += timed(fn[1], 1)
            res['%s_%s_ms_bipartite' % (kind, name)] = [round(t, 3) for t in tb]
            res['%s_%s_ms_union' % (kind, name)] = [round(t, 3) for t in tu]
    res['peak_mem_gb'] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
