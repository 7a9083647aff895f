"""Time a decoder-shaped bipartite NNConv against the same map run as a square conv on the union graph (DESIGN 4.10):

    python scripts/bipartite_probe.py [--reps 5] [--precision f16]

Sources: the 121 x 121 mesh of [0, 1]^2; targets: the 241 x 241 query points; an edge joins every source within
r = 0.05 of a target.  Edge attributes (x_src, x_dst, a_src, a_dst) as the reference builds them; width 64 on both
sides, edge network DenseNet([6, 512, 1024, 64 * 64]) (ker_width 1024), aggr='mean'.  For each form: one forward
(under no_grad, edge features cached as a trained GKN evaluates) and one training step (forward + backward through
x_src, x_dst, edge_attr and every parameter, edge features rebuilt each step).  The two forms alternate within one
process, so the spread between repetitions is measured beside the difference.  Prints one JSON line.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def mesh(n):
    t = torch.linspace(0, 1, n, dtype=torch.float64)
    return torch.stack(torch.meshgrid(t, t, indexing='ij'), -1).view(-1, 2)


def ball_edges(src_pos, dst_pos, r, chunk=4096):
    """(src, dst) with |src_pos - dst_pos| <= r, grouped by target."""
    out = []
    for d0 in range(0, dst_pos.size(0), chunk):
        d = torch.cdist(dst_pos[d0:d0 + chunk], src_pos)
        di, si = torch.nonzero(d <= r, as_tuple=True)
        out.append(torch.stack([si, di + d0]))
    return torch.cat(out, 1)


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--precision', default='f16')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bipartite_probe: no CUDA device (timings are GPU-only)')
    from graph_pde_b200.nn_conv import NNConv_old
    from tests.helpers import DenseNetLike
    dev = 'cuda'
    ps, pd = mesh(121).to(dev), mesh(241).to(dev)
    ns, nd = ps.size(0), pd.size(0)
    ei = ball_edges(ps, pd, 0.05)
    g = torch.Generator(device=dev).manual_seed(0)
    a_s, a_d = torch.rand(ns, 1, device=dev, generator=g), torch.rand(nd, 1, device=dev, generator=g)
    ea = torch.cat([ps[ei[0]].float(), pd[ei[1]].float(), a_s[ei[0]], a_d[ei[1]]], 1)
    union = torch.stack([ei[0], ei[1] + ns])
    xs = torch.randn(ns, 64, device=dev, generator=g)
    xd = torch.randn(nd, 64, device=dev, generator=g)
    xu = torch.cat([xs, xd])
    gd = torch.randn(nd, 64, device=dev, generator=g)
    torch.manual_seed(0)
    conv = NNConv_old(64, 64, DenseNetLike([6, 512, 1024, 64 * 64]), aggr='mean', precision=args.precision).to(dev)

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

    diff = float((fwd_bip() - fwd_union()).abs().max() / fwd_union().abs().max())
    res = {'card': torch.cuda.get_device_name(0), 'n_src': ns, 'n_dst': nd, 'edges': int(ei.size(1)),
           'precision': args.precision, 'rel_diff_bip_vs_union': diff}
    for name, fn in (('forward', (fwd_bip, fwd_union)), ('train_step', (step_bip, step_union))):
        for f in fn:
            f()                               # warm-up: plans, edge features, workspaces
        tb, tu = [], []
        for _ in range(args.reps):            # alternate the two forms
            tb += timed(fn[0], 1)
            tu += timed(fn[1], 1)
        res[name + '_ms_bipartite'] = [round(t, 3) for t in tb]
        res[name + '_ms_union'] = [round(t, 3) for t in tu]
    res['peak_mem_gb'] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
