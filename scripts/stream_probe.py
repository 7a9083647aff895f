"""Partially resident (streamed) edge features at full size: time per conv-stack step and parity.

    python scripts/stream_probe.py [--steps N] [--s301]

1. darcy 241^2, r=0.05, w=64, ker_width=1024, T=6 at precision f16x2 (its edge features, 4 KB per edge, do not fit an
   80 GB card): the automatic policy (allocation fails -> a resident prefix sized from the free memory), ms per step,
   E_res and chunks per application, and max|out-ref|/max|ref| against the edge-chunked fp32 reference ops on the GPU.
2. the same graph at f16 with the cache budget at all / 24 GB / 0: the cost of recomputing the streamed part.
3. with --s301: a 301^2 mesh (about 6e7 edges) at f16, automatic policy, with parity.

A "step" is the T applications of the shared conv with the resident prefix already cached; the first step, which also
computes the prefix, is reported separately.  Prints the device and its power limit."""
import argparse
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)
from graph_pde_b200 import graphs, nn_conv  # noqa: E402
from graph_pde_b200.nn_conv import NNConv_old, _Streamed  # noqa: E402
from oracle import nnconv_oracle as O  # noqa: E402
from tests.helpers import make_conv, oracle_stack_on_cuda, rel_err  # noqa: E402


def _power_limit():
    try:
        res = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'], stdout=subprocess.PIPE,
                             stderr=subprocess.STDOUT, text=True, timeout=30)
        return res.stdout.strip().splitlines()[0] if res.returncode == 0 else 'unknown (nvidia-smi failed)'
    except (OSError, subprocess.SubprocessError, IndexError):
        return 'unknown (nvidia-smi not available)'


def _case(s, r, dev, w=64, kw=1024, seed=3):
    ei = graphs.ball_connectivity(s, r, dev, True)
    _, _, ea = graphs.darcy_sample(s, r, dev, seed=seed, edge_index=ei)
    ws, bs, root, bias = O.reference_init(w, w, [6, kw, kw, w * w], seed=0)
    torch.manual_seed(seed)
    return ei, ea, torch.randn(s * s, w, device=dev), ws, bs, root, bias


def _stack(conv, x, ei, ea, T):
    with torch.no_grad():
        for _ in range(T):
            x = torch.relu(conv(x, ei, ea))
    return x


def _run(conv, x0, ei, ea, T, steps):
    """(first-step ms, median steady-step ms, output, streaming info)."""
    conv.invalidate()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = _stack(conv, x0, ei, ea, T)
    torch.cuda.synchronize()
    first = (time.perf_counter() - t0) * 1e3
    ms = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = _stack(conv, x0, ei, ea, T)
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    ent = next(iter(conv._h_cache.values()))[0]
    info = dict(E_res=ent.E_res, chunks=ent.n_chunks, resident_GB=ent.h_res.numel() / 1e9) if isinstance(ent, _Streamed) \
        else dict(E_res=ei.size(1), chunks=0, resident_GB=ent.numel() / 1e9)
    return first, sorted(ms)[len(ms) // 2], out, info


def _parity(conv, out, x0, ei, ea, ws, bs, root, bias, T, dev):
    conv.invalidate()
    torch.cuda.empty_cache()
    ref = oracle_stack_on_cuda(x0, ei, ea, [v.to(dev) for v in ws], [v.to(dev) for v in bs], root.to(dev), bias.to(dev), T,
                               edge_chunk=1 << 16)
    return rel_err(out, ref[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=2)
    ap.add_argument('--s301', action='store_true')
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    T = 6
    print('device: %s, power limit: %s' % (torch.cuda.get_device_name(dev), _power_limit()))
    ei, ea, x0, ws, bs, root, bias = _case(241, 0.05, dev)
    E = ei.size(1)
    print('darcy241: E=%d, T=%d, width=64, ker_width=1024' % (E, T))

    conv = make_conv(NNConv_old, ws, bs, root, bias, 'mean', 64, 64, 'f16x2', dev)
    first, ms, out, info = _run(conv, x0, ei, ea, T, args.steps)
    err = _parity(conv, out, x0, ei, ea, ws, bs, root, bias, T, dev)
    print('f16x2 auto: first step %.0f ms, step %.0f ms (%.3g edge-apps/s), E_res=%d (%.1f%%, %.1f GB), %d chunks per '
          'application, max|out-ref|/max|ref| = %.2e (bound 2e-5)' % (first, ms, E * T / (ms * 1e-3), info['E_res'],
                                                                     100.0 * info['E_res'] / E, info['resident_GB'],
                                                                     info['chunks'], err))
    del conv, out
    torch.cuda.empty_cache()

    conv = make_conv(NNConv_old, ws, bs, root, bias, 'mean', 64, 64, 'f16', dev)
    for name, budget in (('all', None), ('24GB', 24 << 30), ('0', 0)):
        conv.edge_feature_bytes = budget
        first, ms, out, info = _run(conv, x0, ei, ea, T, args.steps)
        print('f16 budget %s: first step %.0f ms, step %.0f ms (%.3g edge-apps/s), E_res=%d (%.1f%%), %d chunks per '
              'application' % (name, first, ms, E * T / (ms * 1e-3), info['E_res'], 100.0 * info['E_res'] / E,
                               info['chunks']))
    del conv, out, ei, ea
    torch.cuda.empty_cache()

    if args.s301:
        ei, ea, x0, ws, bs, root, bias = _case(301, 0.05, dev)
        E = ei.size(1)
        conv = make_conv(NNConv_old, ws, bs, root, bias, 'mean', 64, 64, 'f16', dev)
        first, ms, out, info = _run(conv, x0, ei, ea, T, 1)
        err = _parity(conv, out, x0, ei, ea, ws, bs, root, bias, T, dev)
        print('darcy301 f16 auto: E=%d, first step %.0f ms, step %.0f ms, E_res=%d (%.1f%%), %d chunks per application, '
              'max|out-ref|/max|ref| = %.2e (bound 2e-3)' % (E, first, ms, info['E_res'], 100.0 * info['E_res'] / E,
                                                             info['chunks'], err))
    print('streamed chunk passes: %d' % nn_conv.stats['streamed_chunk_passes'])


if __name__ == '__main__':
    main()
