"""Write tests/golden/g11_gaussian_nnconv.npz by running the reference's own graph-neural-operator/nn_conv.py class
NNConv_Gaussian, unmodified, over oracle/pyg_stub on the CPU:

    python scripts/gen_golden_gauss.py /path/to/graph-pde        # a checkout of neuraloperator/graph-pde

Cases: aggr add / mean / max, with and without root and bias; nn is Linear(1, 64) in half of them and
Sequential(Linear(1, 16), ReLU(), Linear(16, 64)) in the other half.  The graph has duplicate edges (with their own
attributes), nodes without in-edges and nodes without out-edges.  Each case stores the module's state dict after its
seeded construction (the reference's init stream), its output, and the reference's autograd gradients of the loss
sum(out * gw) w.r.t. x, edge_attr and every parameter.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import golden  # noqa: E402


def main(ref_root):
    sys.path[:0] = [os.path.join(ROOT, 'oracle', 'pyg_stub'), os.path.join(ref_root, 'graph-neural-operator')]
    import nn_conv            # the reference module, unmodified
    g = torch.Generator().manual_seed(11)
    N, E, C, kin = 30, 240, 64, 6
    src = torch.randint(0, N - 4, (E,), generator=g)     # last 4 nodes: no out-edges
    dst = torch.randint(2, N, (E,), generator=g)         # first 2 nodes: no in-edges
    src[5:12], dst[5:12] = src[0], dst[0]                 # duplicate edges
    ei = torch.stack([src, dst])
    sign = torch.where(torch.rand(E, kin, generator=g) < 0.5, -1.0, 1.0)
    ea = (torch.rand(E, kin, generator=g) + 0.25) * sign   # |p1 p2| >= 1/16: finite amplitudes
    x = torch.randn(N, C, generator=g)
    gw = torch.randn(N, C, generator=g)                  # loss = sum(out * gw)
    rec = dict(edge_index=ei.numpy().astype(np.int64), edge_attr=ea.numpy(), x=x.numpy(), gw=gw.numpy())
    cases = []
    for aggr in ('add', 'mean', 'max'):
        for rw in (True, False):
            for bs in (True, False):
                cases.append((aggr, rw, bs, 'linear' if (rw == bs) else 'mlp'))
    for i, (aggr, rw, bs, net) in enumerate(cases):
        torch.manual_seed(200 + i)
        if net == 'linear':
            mlp = torch.nn.Linear(1, C)
        else:
            mlp = torch.nn.Sequential(torch.nn.Linear(1, 16), torch.nn.ReLU(), torch.nn.Linear(16, C))
        conv = nn_conv.NNConv_Gaussian(C, C, mlp, aggr=aggr, root_weight=rw, bias=bs)
        p = 'c%d_' % i
        rec[p + 'case'] = np.array([aggr, str(rw), str(bs), net])
        rec[p + 'repr'] = np.array(repr(conv))
        rec[p + 'keys'] = np.array(list(conv.state_dict().keys()))
        for k, v in conv.state_dict().items():
            rec[p + 'sd_' + k] = v.numpy().copy()
        xg, eag = x.clone().requires_grad_(), ea.clone().requires_grad_()
        out = conv(xg, ei, eag)
        (out * gw).sum().backward()
        rec[p + 'out'] = out.detach().numpy()
        rec[p + 'grad_x'] = xg.grad.numpy()
        rec[p + 'grad_edge_attr'] = eag.grad.numpy()
        for k, v in conv.named_parameters():
            rec[p + 'grad_' + k] = v.grad.numpy()
    rec['n_cases'] = np.array(len(cases))
    golden.save(os.path.join(ROOT, 'tests', 'golden', 'g11_gaussian_nnconv.npz'), **rec)
    print('wrote g11_gaussian_nnconv.npz: %d cases' % len(cases))


if __name__ == '__main__':
    main(sys.argv[1])
