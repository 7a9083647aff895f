#!/usr/bin/env python
"""Time the wgmma GEMM alone (CUDA events) at the edge-MLP chunk shape for several K, next to a pure
write (memset), a copy of the same output size and the same product through torch.mm (cuBLAS, fp16) as the
yardstick: separates 'epilogue/store bound' from 'DRAM write bound'.  The last lines run the product's real
configuration, the edge-feature pass of a ker_width-1024 conv (overflow check on, bias and ReLU, chunk-major
output at the edge-feature chunk shape), and report its per-chunk kernel times."""
import ctypes
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
from graph_pde_b200 import _lib  # noqa: E402


def timed(fn, reps=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e3   # us


def main():
    L = _lib.lib()
    dev = torch.device('cuda:0')
    M, N = int(os.environ.get('PROBE_M', 253184)), 1024
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    C = torch.empty(M, N, dtype=torch.float16, device=dev)
    C2 = torch.empty_like(C)
    bias = torch.randn(N, device=dev)
    out_mb = C.numel() * 2 / 1e6
    print('output %.0f MB' % out_mb)
    t = timed(lambda: C.zero_())
    print('memset          %8.1f us  %6.0f GB/s written' % (t, out_mb / t * 1e3))
    t = timed(lambda: C2.copy_(C))
    print('copy            %8.1f us  %6.0f GB/s (r+w)' % (t, 2 * out_mb / t * 1e3))
    for K in (64, 128, 256, 512, 1024):
        A = (torch.randn(M, K, device=dev) * 0.5).half()
        B = (torch.randn(N, K, device=dev) * 0.5).half()
        for relu, b in ((1, None), (1, bias)):
            def run():
                _lib.check(L.nnconv_gemm_16b(_lib.PREC['f16'], ctypes.c_void_p(A.data_ptr()), M, K,
                                             ctypes.c_void_p(B.data_ptr()), N,
                                             ctypes.c_void_p(b.data_ptr() if b is not None else 0), relu,
                                             ctypes.c_void_p(C.data_ptr()), st))
            t = timed(run)
            print('gemm K=%4d bias=%d %8.1f us  %6.0f GB/s written  %7.1f TFLOP/s' %
                  (K, b is not None, t, out_mb / t * 1e3, 2.0 * M * N * K / t / 1e6))
        t = timed(lambda: torch.mm(A, B.t(), out=C))
        print('cublas K=%4d      %8.1f us  %6.0f GB/s written  %7.1f TFLOP/s' %
              (K, t, out_mb / t * 1e3, 2.0 * M * N * K / t / 1e6))
        del A, B
    del C, C2
    edge_feature_pass(L, dev)


def edge_feature_pass(L, dev, chunks=4, width=64, ker_width=1024):
    """nnconv_edge_features over `chunks` edge-feature chunks of the default workspace (the rows one chunk of the
    241x241 Darcy graph has), timed per kernel kind with the library's profiler."""
    from graph_pde_b200 import nn_conv
    torch.manual_seed(0)
    n_nodes, rows = 58081, 508288
    E = chunks * rows
    ei = torch.randint(0, n_nodes, (2, E), device=dev)
    ea = torch.rand(E, 6, device=dev)
    mlp = torch.nn.Sequential(torch.nn.Linear(6, ker_width), torch.nn.ReLU(), torch.nn.Linear(ker_width, ker_width),
                              torch.nn.ReLU(), torch.nn.Linear(ker_width, width * width))
    conv = nn_conv.NNConv_old(width, width, mlp, aggr='mean').to(dev)
    plan = nn_conv.get_plan(ei, n_nodes)
    prepared = conv._get_prepared('f16')
    for _ in range(2):
        conv._h_cache.clear()
        conv.edge_features(plan, prepared, ea)
    torch.cuda.synchronize()
    reps = 3
    _lib.check(L.nnconv_profile_begin())
    for _ in range(reps):
        conv._h_cache.clear()
        conv.edge_features(plan, prepared, ea)
    ms_k = (ctypes.c_double * 8)()
    n_k = (ctypes.c_int64 * 8)()
    _lib.check(L.nnconv_profile_end(ms_k, n_k, 8))
    for k, name in ((0, 'edge_layer1'), (1, 'hidden_gemm')):
        per = ms_k[k] * 1e3 / max(1, n_k[k])
        print('%-11s E=%d: %d launches, %8.1f us per launch' % (name, E, n_k[k], per))


if __name__ == '__main__':
    main()
