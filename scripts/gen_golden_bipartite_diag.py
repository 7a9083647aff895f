"""Write tests/golden/g13_bipartite_channelwise.npz by running the reference's own graph-neural-operator/nn_conv.py
classes NNConv (the diagonal kernel) and NNConv_Gaussian, unmodified, over oracle/pyg_stub on the CPU, on the union
graph of a bipartite map:

    python scripts/gen_golden_bipartite_diag.py /path/to/graph-pde        # a checkout of neuraloperator/graph-pde

The reference has no bipartite input, so each case runs it on the union node set [x_src; x_dst] with the edges
(src, N_src + dst) and keeps the output rows [N_src:], which is the bipartite map.  Sources [N_src - 3, N_src) have no
out-edges and targets [0, 2) no in-edges.  Cases, for each conv: N_src > N_dst and N_src < N_dst at aggr add, mean and
max with root and bias, and one add case without them.  Each case stores the module's state dict after its seeded
construction, the output, and the reference's autograd gradients of sum(out * gw) w.r.t. x_src, x_dst, edge_attr and
every parameter.  The diagonal conv runs at C = 8 with nn = Linear(3, 16), ReLU, Linear(16, 8); the Gaussian one at
C = 64 (the reference hard-codes it) with nn = Linear(1, 64).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import golden  # noqa: E402

# (conv, N_src, N_dst, E, aggr, root_weight and bias)
CASES = [(conv, n_src, n_dst, e, aggr, True) for conv in ('diag', 'gauss')
         for n_src, n_dst, e in ((40, 17, 220), (13, 36, 180)) for aggr in ('add', 'mean', 'max')]
CASES += [('diag', 13, 36, 180, 'add', False), ('gauss', 40, 17, 220, 'add', False)]


def main(ref_root):
    sys.path[:0] = [os.path.join(ROOT, 'oracle', 'pyg_stub'), os.path.join(ref_root, 'graph-neural-operator')]
    import nn_conv            # the reference module, unmodified
    kin = 3
    rec = {}
    for i, (kind, n_src, n_dst, E, aggr, rb) in enumerate(CASES):
        C = 8 if kind == 'diag' else 64
        g = torch.Generator().manual_seed(130 + i)
        src = torch.randint(0, n_src - 3, (E,), generator=g)
        dst = torch.randint(2, n_dst, (E,), generator=g)
        sign = torch.where(torch.rand(E, kin, generator=g) < 0.5, -1.0, 1.0)
        ea = (torch.rand(E, kin, generator=g) + 0.25) * sign      # |p1 p2| >= 1/16: finite Gaussian amplitudes
        x_src = torch.randn(n_src, C, generator=g)
        x_dst = torch.randn(n_dst, C, generator=g)
        gw = torch.randn(n_dst, C, generator=g)
        torch.manual_seed(3000 + i)
        if kind == 'diag':
            mlp = torch.nn.Sequential(torch.nn.Linear(kin, 16), torch.nn.ReLU(), torch.nn.Linear(16, C))
            conv = nn_conv.NNConv(C, C, mlp, aggr=aggr, root_weight=rb, bias=rb)
        else:
            conv = nn_conv.NNConv_Gaussian(C, C, torch.nn.Linear(1, C), aggr=aggr, root_weight=rb, bias=rb)
        pre = 'c%d_' % i
        rec[pre + 'case'] = np.array([kind, aggr, str(n_src), str(n_dst), str(rb)])
        for k, v in conv.state_dict().items():
            rec[pre + 'sd_' + k] = v.numpy().copy()
        xs, xd, eag = x_src.clone().requires_grad_(), x_dst.clone().requires_grad_(), ea.clone().requires_grad_()
        out = conv(torch.cat([xs, xd]), torch.stack([src, n_src + dst]), eag)[n_src:]
        (out * gw).sum().backward()
        rec[pre + 'edge_index'] = torch.stack([src, dst]).numpy().astype(np.int64)
        rec[pre + 'edge_attr'] = ea.numpy()
        rec[pre + 'x_src'] = x_src.numpy()
        rec[pre + 'x_dst'] = x_dst.numpy()
        rec[pre + 'gw'] = gw.numpy()
        rec[pre + 'out'] = out.detach().numpy()
        rec[pre + 'grad_x_src'] = xs.grad.numpy()
        rec[pre + 'grad_x_dst'] = xd.grad.numpy()
        rec[pre + 'grad_edge_attr'] = eag.grad.numpy()
        for k, v in conv.named_parameters():
            rec[pre + 'grad_' + k] = v.grad.numpy()
    rec['n_cases'] = np.array(len(CASES))
    golden.save(os.path.join(ROOT, 'tests', 'golden', 'g13_bipartite_channelwise.npz'), **rec)
    print('wrote g13_bipartite_channelwise.npz: %d cases' % len(CASES))


if __name__ == '__main__':
    main(sys.argv[1])
