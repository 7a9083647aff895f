"""Write tests/golden/g8_diag_nnconv.npz by running the reference's own graph-neural-operator/nn_conv.py class NNConv
(the diagonal-kernel conv), unmodified, over oracle/pyg_stub on the CPU:

    python scripts/gen_golden_diag.py /path/to/graph-pde        # a checkout of neuraloperator/graph-pde

Cases: aggr add / mean / max, with and without root and bias, and one 1-D x (in = out = 1).  Each case stores the
module's state dict after its seeded construction (the reference's init stream) and its output.
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
    g = torch.Generator().manual_seed(8)
    N, E, C, kin, width = 30, 240, 64, 3, 64
    src = torch.randint(0, N - 4, (E,), generator=g)     # last 4 nodes: no out-edges
    dst = torch.randint(2, N, (E,), generator=g)         # first 2 nodes: no in-edges
    src[5:12], dst[5:12] = src[0], dst[0]                 # duplicate edges
    ei = torch.stack([src, dst])
    ea = torch.randn(E, kin, generator=g)
    x = torch.randn(N, C, generator=g)
    x1 = torch.randn(N, generator=g)
    rec = dict(edge_index=ei.numpy().astype(np.int64), edge_attr=ea.numpy(), x=x.numpy(), x1=x1.numpy())
    cases = []
    for aggr in ('add', 'mean', 'max'):
        for rw in (True, False):
            for bs in (True, False):
                cases.append((aggr, rw, bs, C))
    cases.append(('mean', True, True, 1))
    for i, (aggr, rw, bs, c) in enumerate(cases):
        torch.manual_seed(100 + i)
        mlp = torch.nn.Sequential(torch.nn.Linear(kin, width), torch.nn.ReLU(), torch.nn.Linear(width, c))
        conv = nn_conv.NNConv(c, c, mlp, aggr=aggr, root_weight=rw, bias=bs)
        with torch.no_grad():
            out = conv(x if c == C else x1, ei, ea)
        p = 'c%d_' % i
        rec[p + 'case'] = np.array([aggr, str(rw), str(bs), str(c)])
        rec[p + 'repr'] = np.array(repr(conv))
        rec[p + 'keys'] = np.array(list(conv.state_dict().keys()))
        for k, v in conv.state_dict().items():
            rec[p + 'sd_' + k] = v.numpy().copy()
        rec[p + 'out'] = out.numpy()
    rec['n_cases'] = np.array(len(cases))
    golden.save(os.path.join(ROOT, 'tests', 'golden', 'g8_diag_nnconv.npz'), **rec)
    print('wrote g8_diag_nnconv.npz: %d cases' % len(cases))


if __name__ == '__main__':
    main(sys.argv[1])
