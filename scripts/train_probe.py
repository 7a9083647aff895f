#!/usr/bin/env python
"""One training step (forward + tensor-core backward + Adam) of KernelNN on a synthetic Darcy graph, bracketed by
cudaProfilerStart/Stop so that `ncu --profile-from-start off` sees exactly one step:

    ncu --metrics gpu__time_duration.sum --clock-control none --profile-from-start off --csv \
        --log-file gpurun_out/train_launches.csv python scripts/train_probe.py [darcy241|darcy85]
Without ncu it prints the CUDA-event time of the step (the median of --rounds steps), the device and its power limit.

    python scripts/train_probe.py darcy85 --precision f16x2 [--backward fp32] [--rounds N] [--kernels]
selects the operand precision of the step and pins the backward to the fp32 CUDA-core path (--backward fp32; the
default 'auto' takes the tensor-core backward where it covers the shapes); --kernels adds a torch.profiler table of
the per-kernel CUDA times of one step.

    python scripts/train_probe.py [darcy241|darcy301] --precision f16x2 --edge-feature-bytes auto|N
trains on streamed edge features (streamed_training=True): N bounds the cached prefix of h to N bytes, 'auto' keeps the
whole h when it fits and otherwise the prefix the free device memory allows beside the backward's workspace.  Prints
the resident fraction of the edges and the chunks per forward and per backward application besides the step time.

    python scripts/train_probe.py [darcy241|darcy85] --edge-attr-grad [--rounds N]
times the same step with edge_attr built from a coefficient field theta by graphs.ball_edge_attr, once with theta a
plain tensor and once with theta a leaf that requires grad (so that the step also delivers d loss / d edge_attr and
d loss / d theta), alternating the two in one run, and prints both median step times, the device and its power limit."""
import argparse
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)
from bench import WORKLOADS  # noqa: E402
from graph_pde_b200 import graphs  # noqa: E402
from graph_pde_b200.models import KernelNN  # noqa: E402


class _Data(object):
    pass


# + a mesh finer than the headline one, whose f16 edge features (about 117 GiB) do not fit an 80 GB card
_WORKLOADS = dict(WORKLOADS, darcy301=dict(s=301, r=0.05, width=64, ker_width=1024, depth=6))


def _power_limit():
    try:
        res = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'], stdout=subprocess.PIPE,
                             stderr=subprocess.STDOUT, text=True, timeout=30)
        return res.stdout.strip().splitlines()[0] if res.returncode == 0 else 'unknown (nvidia-smi failed)'
    except (OSError, subprocess.SubprocessError, IndexError):
        return 'unknown (nvidia-smi not available)'


def _timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def _print_streaming(conv, nn_conv, T):
    """Resident fraction and chunk counts of the streamed edge features of the last step (or 'whole h')."""
    import ctypes
    from graph_pde_b200 import _lib
    st = next((v[0] for v in conv._h_cache.values()), None)
    if st is None:
        st = getattr(getattr(conv, '_tstate', None), 'h', None)
    if not isinstance(st, nn_conv._Streamed):
        print('edge features: whole h resident (no streaming)')
        return
    plan, prep = conv._tstate.plan, conv._tstate.prepared
    b = ctypes.c_size_t()
    if st.bwd_ws is not None:             # the tensor-core backward's workspace, allocated with the prefix
        ws_apply = ws_mlp = st.bwd_ws.numel()
    else:
        _lib.check(_lib.lib().nnconv_backward_apply_streamed_sizes(plan.handle, prep.handle, st.E_res,
                                                                   nn_conv._BWD_APPLY_WS_BYTES, nn_conv._EF_WS_BYTES,
                                                                   ctypes.byref(b)))
        ws_apply = b.value
        _lib.check(_lib.lib().nnconv_backward_mlp_streamed_sizes(plan.handle, prep.handle, st.E_res, T,
                                                                 nn_conv._BWD_MLP_WS_BYTES, ctypes.byref(b)))
        ws_mlp = b.value
    bwd = nn_conv._streamed_chunks(plan, prep, st.E_res, 0, ws_apply)
    mlp = nn_conv._streamed_chunks(plan, prep, st.E_res, T, ws_mlp)
    print('edge features: resident %d of %d edges (%.1f %%), %.1f GiB; chunks per forward application %d, per backward '
          'application %d, MLP pass %d' % (st.E_res, plan.E, 100.0 * st.E_res / max(plan.E, 1), st.h_res.numel() / 2 ** 30,
                                          st.n_chunks, bwd, mlp))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('workload', nargs='?', default='darcy241', choices=sorted(_WORKLOADS))
    ap.add_argument('--edge-attr-grad', action='store_true')
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--precision', default='f16', choices=['f16', 'bf16', 'f16x2'])
    ap.add_argument('--backward', default='auto', choices=['auto', 'fp32'])
    ap.add_argument('--kernels', action='store_true')
    ap.add_argument('--edge-feature-bytes', default=None, help="N or 'auto': train on streamed edge features")
    args = ap.parse_args()
    from graph_pde_b200 import nn_conv
    nn_conv._BWD_MODE = args.backward
    cfg = _WORKLOADS[args.workload]
    dev = torch.device('cuda:0')
    s, r, w, kw, T = cfg['s'], cfg['r'], cfg['width'], cfg['ker_width'], cfg['depth']
    torch.manual_seed(0)
    model = KernelNN(w, kw, T, 6, in_width=6, precision=args.precision).to(dev)
    if args.edge_feature_bytes is not None:
        model.conv1.streamed_training = True
        model.conv1.edge_feature_bytes = None if args.edge_feature_bytes == 'auto' else int(args.edge_feature_bytes)
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
        return loss

    if not args.edge_attr_grad:
        step()
        torch.cuda.synchronize()
        torch.cuda.profiler.start()
        times = [_timed(step)]
        torch.cuda.profiler.stop()
        for _ in range(args.rounds - 1):
            times.append(_timed(step))
        n_mlp = nn_conv.stats.get('mlp_backwards', 0)
        print('device: %s, power limit: %s' % (torch.cuda.get_device_name(dev), _power_limit()))
        print('%s: E=%d, T=%d, width=%d, ker_width=%d, precision=%s, backward=%s (tensor-core MLP passes so far: %d)' % (
            args.workload, ei.size(1), T, w, kw, args.precision, args.backward, n_mlp))
        print('training step: median %.2f ms  (all: %s)' % (statistics.median(times), ', '.join('%.2f' % v for v in times)))
        if args.edge_feature_bytes is not None:
            _print_streaming(model.conv1, nn_conv, T)
        if args.kernels:
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                step()
                torch.cuda.synchronize()
            print(prof.key_averages().table(sort_by='cuda_time_total', row_limit=25, max_name_column_width=90))
        return

    # theta = the coefficient column of the node features (darcy_sample: x = [grid, a, ...], edge_attr uses a)
    grid = graphs.square_grid(s, dev)
    theta0 = x6[:, 2].clone()

    def step_theta(need):
        theta = theta0.clone().requires_grad_(need)
        d.edge_attr = graphs.ball_edge_attr(grid, ei, theta)
        step()
        if need:
            assert theta.grad is not None and bool(torch.isfinite(theta.grad).all())

    times = {False: [], True: []}
    for need in (False, True):             # warm-up: both variants, every shape
        step_theta(need)
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for need in (False, True):
            times[need].append(_timed(lambda: step_theta(need)))
    base, with_ea = statistics.median(times[False]), statistics.median(times[True])
    print('device: %s, power limit: %s' % (torch.cuda.get_device_name(dev), _power_limit()))
    print('%s: E=%d, T=%d, width=%d, ker_width=%d, %d alternating rounds' % (args.workload, ei.size(1), T, w, kw,
                                                                              args.rounds))
    print('training step, edge_attr without grad: median %.2f ms  (all: %s)' % (base, ', '.join('%.2f' % v for v in times[False])))
    print('training step, edge_attr with grad:    median %.2f ms  (all: %s)' % (with_ea, ', '.join('%.2f' % v for v in times[True])))
    print('overhead: %.2f ms (%.1f %%)' % (with_ea - base, 100.0 * (with_ea - base) / base))


if __name__ == '__main__':
    main()
