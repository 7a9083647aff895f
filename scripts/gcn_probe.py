"""Times GCNConv on the configuration of the reference's neurips4_GCN.py: the 421^2 grid_edge lattice, six node
features, width 128, ker_width 1024, four convs applied depth = 4 times, batch 1.  For each precision: forward and Adam
training-step time, eager and replayed from a CUDA graph (GraphedForward, GraphedTrainStep); the time of one
application's kernel (k_gcn_tc, or the fp32 path's kernels) with the bytes it has to move and the rate that gives; and the same forward in fp32 torch ops on the GPU (gcn_norm per call, index_add_
aggregation) for comparison.  Prints one JSON object with the card name and power limit read in the same run.

    python scripts/gcn_probe.py [--steps 20] [--precisions f16,bf16,f16x2,fp32] [--out FILE]
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from graph_pde_b200 import GraphedForward, GraphedTrainStep  # noqa: E402
from graph_pde_b200.graphs import grid_edge  # noqa: E402
from graph_pde_b200.models import GCN_Net  # noqa: E402
from scripts.diag_probe import card  # noqa: E402
from tests import gcn_oracle as G  # noqa: E402


def timed(fn, steps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


class Data(object):
    pass


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--precisions', default='f16,bf16,f16x2,fp32')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    dev = torch.device('cuda')
    s, width, ker_width, depth, node_features = 421, 128, 1024, 4, 6
    grid, ei = grid_edge(s, s, device=dev)
    n, e = grid.size(0), ei.size(1)
    a = torch.rand(n, node_features - 2, device=dev)       # the coefficient, its smoothed form, its x and y gradients
    d = Data()
    d.x, d.edge_index = torch.cat([grid, a], 1), ei
    y = torch.randn(n, 1, device=dev)
    name, limit = card()
    res = {'card': name, 'power_limit': limit, 'nodes': n, 'edges': e, 'width': width, 'ker_width': ker_width,
           'depth': depth, 'node_features': node_features}
    # bytes one application must move: x gathered once per node (assuming the lattice's reuse hits L2), out written,
    # both CSR entries (index + norm) and the row pointers
    app_bytes = n * width * 4 * 2 + (e + n) * 8 + n * 4
    res['app_bytes'] = app_bytes
    for prec in args.precisions.split(','):
        torch.manual_seed(0)
        model = GCN_Net(width, ker_width, depth, in_width=node_features, precision=prec).to(dev)
        conv = model.conv1
        x = torch.randn(n, width, device=dev)
        r = {}
        with torch.no_grad():
            r['app_ms'] = timed(lambda: conv(x, ei), args.steps * 4)
            r['app_GBps'] = app_bytes / (r['app_ms'] * 1e-3) / 1e9
            r['forward_ms'] = timed(lambda: model(d), args.steps)
        gf = GraphedForward(model, d)
        r['forward_graphed_ms'] = timed(gf.replay, args.steps)
        del gf
        opt = torch.optim.Adam(model.parameters(), lr=1e-3, capturable=True)

        def step():
            opt.zero_grad(set_to_none=True)
            F.mse_loss(model(d), y).backward()
            opt.step()
        r['train_step_ms'] = timed(step, args.steps)
        g = GraphedTrainStep(lambda xx, yy: F.mse_loss(model(d), yy), model, opt, d.x, y)
        r['train_step_graphed_ms'] = timed(g.replay, args.steps)
        res[prec] = r
    # the same math in fp32 torch ops (PyG's gcn_norm recomputed per call, index_add_ aggregation)
    torch.manual_seed(0)
    W = torch.randn(width, width, device=dev) * 0.1
    b = torch.zeros(width, device=dev)
    x = torch.randn(n, width, device=dev)

    def torch_app():
        src, dst, norm = G.gcn_norm(ei, n, dtype=torch.float32)
        xw = x @ W
        return torch.zeros_like(xw).index_add_(0, dst, norm[:, None] * xw[src]) + b
    with torch.no_grad():
        res['torch_fp32_app_ms'] = timed(torch_app, args.steps * 4)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
