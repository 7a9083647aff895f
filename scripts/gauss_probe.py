"""Times the Gaussian-kernel conv (GaussianNNConv, csrc/gauss.cu) on one card, C = 64, aggr mean:

- one application (k_apply_gauss), one backward (k_bwd_gauss with the sigma and edge_attr gradients), and a training
  step of the conv alone (T = 6 applications with ReLUs, forward and backward through autograd, nn = Linear(1, 64));
- one application of the diagonal-kernel conv (k_apply_diag, d cached) on the same graph;
- the reference's math in torch ops on the GPU (diag_embed into [E, 64, 64], then matmul), where that tensor fits:
  forward, and forward + backward, at 61^2; forward at 85^2.  Checks the two agree.

Meshes: darcy 61^2 and 85^2 at r = 0.10, 241^2 at r = 0.05 (graphs.darcy_sample).  Columns 1 and 2 of its edge_attr are
replaced by |p| + 0.5 so that every amplitude 1 / sqrt(|p1 p2|) is finite.  Prints one JSON object with the card name
and power limit read in the same run.

    python scripts/gauss_probe.py [--steps 20] [--sizes 61,85,241] [--out FILE]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from graph_pde_b200 import GaussianNNConv, graphs  # noqa: E402
from graph_pde_b200.nn_conv import DiagNNConv, _f32, get_plan  # noqa: E402
from scripts.diag_probe import card, ms  # noqa: E402

C = 64
REF_FWD_MAX_EDGES = 2_000_000      # [E, 64, 64] fp32: 32 GB at this edge count
REF_BWD_MAX_EDGES = 500_000        # forward + backward keep about three such tensors


def reference_ops(conv, x, ei, ea):
    """nn_conv.py:174-182 and MessagePassing's mean, in torch ops on the GPU."""
    src, dst = ei
    one = torch.ones(1, device=x.device)
    a = 1 / torch.sqrt(torch.abs(ea[:, 1] * ea[:, 2]))
    b = torch.exp(-1 * (ea[:, 0] ** 2).view(-1, 1) / (conv.nn(one) ** 2).view(1, -1))
    w = torch.diag_embed(a.reshape(-1, 1).repeat(1, C) * b).view(-1, C, C)
    msg = torch.matmul(x[src].unsqueeze(1), w).squeeze(1)
    out = torch.zeros_like(x).index_add_(0, dst, msg)
    cnt = torch.zeros(x.size(0), device=x.device).index_add_(0, dst, torch.ones_like(dst, dtype=x.dtype))
    return out / cnt.clamp(min=1).unsqueeze(-1) + x @ conv.root + conv.bias


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--sizes', default='61,85,241')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device('cuda:0')
    name, limit = card()
    res = {'card': name, 'power_limit': limit, 'channels': C, 'aggr': 'mean', 'cases': {}}
    for s in [int(v) for v in args.sizes.split(',')]:
        r = 0.05 if s == 241 else 0.10
        torch.manual_seed(0)
        _, ei, ea = graphs.darcy_sample(s, r, device=dev)
        ea = ea.clone()
        ea[:, 1:3] = ea[:, 1:3].abs() + 0.5
        e = ei.size(1)
        x = torch.randn(s * s, C, device=dev)
        conv = GaussianNNConv(C, C, torch.nn.Linear(1, C), aggr='mean').to(dev)
        case = {'edges': e}
        with torch.no_grad():
            out = conv(x, ei, ea)
            plan = get_plan(ei, x.size(0))
            sigma = _f32(conv._sigma(dev))
            case['apply_ms'] = round(ms(lambda: conv._apply_impl(plan, x, ea, sigma), args.steps), 3)
            g = torch.randn_like(x)
            case['backward_ms'] = round(ms(lambda: conv._backward_impl(plan, x, ea, sigma, g, None, True, True),
                                           args.steps), 3)
            # bytes one application must move at least: x_src rows, three attributes and the destination index per
            # edge, out read-modify-written once per node
            case['apply_gb_per_s_lower_bound'] = round((e * (3 * 4 + 4 + 4) + 2 * x.numel() * 4) /
                                                       case['apply_ms'] / 1e6, 1)
            mlp = torch.nn.Sequential(torch.nn.Linear(ea.size(1), 64), torch.nn.ReLU(), torch.nn.Linear(64, C))
            diag = DiagNNConv(C, C, mlp, aggr='mean', precision='fp32').to(dev)
            diag(x, ei, ea)
            feats = diag._features(plan, _f32(ea))
            case['diag_apply_ms'] = round(ms(lambda: diag._apply_impl(plan, feats, x), args.steps), 3)
            del diag, feats
            if e <= REF_FWD_MAX_EDGES:
                ref = reference_ops(conv, x, ei, ea)
                case['reference_ops_forward_ms'] = round(ms(lambda: reference_ops(conv, x, ei, ea), 2), 3)
                case['max_rel_err_vs_reference_ops'] = ((out - ref).abs().max() / ref.abs().max()).item()
                del ref
                torch.cuda.empty_cache()

        def train_step():
            h = x.requires_grad_(True)
            for _ in range(6):
                h = torch.relu(conv(h, ei, ea))
            h.sum().backward()
            x.grad = None
            conv.zero_grad(set_to_none=True)
        case['train_step_T6_ms'] = round(ms(train_step, max(1, args.steps // 4)), 3)
        x.requires_grad_(False)
        if e <= REF_BWD_MAX_EDGES:
            def ref_step():
                xr = x.detach().requires_grad_(True)
                reference_ops(conv, xr, ei, ea).sum().backward()
                conv.zero_grad(set_to_none=True)

            def our_step():
                xr = x.detach().requires_grad_(True)
                conv(xr, ei, ea).sum().backward()
                conv.zero_grad(set_to_none=True)
            case['reference_ops_fwd_bwd_ms'] = round(ms(ref_step, 2), 3)
            case['fwd_bwd_ms'] = round(ms(our_step, args.steps), 3)
            torch.cuda.reset_peak_memory_stats(dev)
            base = torch.cuda.memory_allocated(dev)
            ref_step()
            torch.cuda.synchronize()
            case['reference_ops_fwd_bwd_peak_rise_gb'] = round((torch.cuda.max_memory_allocated(dev) - base) / 1e9, 2)
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        train_step()
        torch.cuda.synchronize()
        case['train_step_T6_peak_rise_gb'] = round((torch.cuda.max_memory_allocated(dev) - base) / 1e9, 3)
        res['cases']['%d' % s] = case
        del ei, ea, conv, out, x
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
