"""Times the diagonal-kernel conv (DiagNNConv, formulation D) on one card: the d build (edge network + last Linear,
chunked) and one application, at 85^2 (r = 0.10) and 241^2 (r = 0.05), width 64, ker_width 1024, f16, against the same
math in fp32 torch ops on the GPU (the edge network over 2^20-edge chunks, then x_src * d and index_add_).  Checks
the two agree.  Also times a training step of the conv alone: T = 6 applications with ReLUs, forward and backward, d
rebuilt as after every optimiser step (the backward's CUDA-core pass through the edge network dominates it).  Prints one
JSON object with the card name and power limit read in the same run.

    python scripts/diag_probe.py [--steps 10] [--sizes 85,241] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from graph_pde_b200 import graphs  # noqa: E402
from graph_pde_b200.nn_conv import DiagNNConv  # noqa: E402


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [v.strip() for v in q.split(',')]
        return name, limit
    except Exception as e:
        return torch.cuda.get_device_name(), 'unknown (%s)' % type(e).__name__


def ms(fn, steps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def torch_ops(conv, x, ei, ea, chunk=1 << 20):
    lin = [m for m in conv.nn if isinstance(m, torch.nn.Linear)]
    src, dst = ei
    d = torch.empty(ea.size(0), conv.out_channels, device=x.device)
    for s in range(0, ea.size(0), chunk):
        h = ea[s:s + chunk]
        for i, l in enumerate(lin):
            h = torch.nn.functional.linear(h, l.weight, l.bias)
            if i < len(lin) - 1:
                h = torch.relu(h)
        d[s:s + chunk] = h
    out = torch.zeros_like(x).index_add_(0, dst, x[src] * d)
    cnt = torch.zeros(x.size(0), device=x.device).index_add_(0, dst, torch.ones_like(dst, dtype=x.dtype))
    return out / cnt.clamp(min=1).unsqueeze(-1) + x @ conv.root + conv.bias, d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--sizes', default='85,241')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device('cuda:0')
    name, limit = card()
    res = {'card': name, 'power_limit': limit, 'precision': 'f16', 'width': 64, 'ker_width': 1024, 'cases': {}}
    for s in [int(v) for v in args.sizes.split(',')]:
        r = 0.10 if s == 85 else 0.05
        torch.manual_seed(0)
        _, ei, ea = graphs.darcy_sample(s, r, device=dev)
        x = torch.randn(s * s, 64, device=dev)
        mlp = torch.nn.Sequential(torch.nn.Linear(ea.size(1), 1024), torch.nn.ReLU(), torch.nn.Linear(1024, 1024),
                                  torch.nn.ReLU(), torch.nn.Linear(1024, 64))
        conv = DiagNNConv(64, 64, mlp, aggr='mean', precision='f16').to(dev)
        with torch.no_grad():
            out = conv(x, ei, ea)
            build = ms(lambda: (conv.invalidate(), conv(x, ei, ea)), max(1, args.steps // 2))
            apply_ms = ms(lambda: conv(x, ei, ea), args.steps)          # d cached: one application
            ref, _ = torch_ops(conv, x, ei, ea)
            torch.cuda.synchronize()
            ref_ms = ms(lambda: torch_ops(conv, x, ei, ea), 1)
        conv.requires_grad_(True)

        def train_step():
            conv.invalidate()
            h = x.requires_grad_(True)
            for _ in range(6):
                h = torch.relu(conv(h, ei, ea))
            h.sum().backward()
            x.grad = None
            conv.zero_grad(set_to_none=True)
        train_ms = ms(train_step, 1)
        x.requires_grad_(False)
        e = ei.size(1)
        res['cases']['%d' % s] = {
            'train_step_T6_ms': round(train_ms, 1),
            'edges': e, 'build_plus_apply_ms': round(build, 3), 'apply_ms': round(apply_ms, 3),
            'build_ms': round(build - apply_ms, 3),
            'apply_gb_per_s': round(e * (4 * 64 + 4) / apply_ms / 1e6, 1),
            'torch_ops_ms': round(ref_ms, 3),
            'max_rel_err_vs_torch_ops': ((out - ref).abs().max() / ref.abs().max()).item()}
        del ei, ea, conv, out, ref
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
