"""Write tests/golden/g12_bipartite_nnconv.npz by running the reference's own NNConv_old
(graph-neural-operator/nn_conv.py) and DenseNet (graph-neural-operator/utilities.py:201-227), unmodified, over
oracle/pyg_stub on the CPU, on the union graph of a bipartite map:

    python scripts/gen_golden_bipartite.py /path/to/graph-pde        # a checkout of neuraloperator/graph-pde

The reference has no bipartite input, so each case runs it on the union node set [x_src; x_dst] with the edges
(src, N_src + dst) and keeps the output rows [N_src:], which is the bipartite map (in_src == in_dst).  Sources
[N_src - 3, N_src) have no out-edges and targets [0, 2) no in-edges.  Cases: N_src > N_dst and N_src < N_dst, each at
aggr add and mean, with root and bias, and one add case without them.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import golden  # noqa: E402

# (N_src, N_dst, E, aggr, root_weight and bias)
CASES = [(40, 17, 220, 'add', True), (40, 17, 220, 'mean', True), (13, 36, 180, 'add', True),
         (13, 36, 180, 'mean', True), (13, 36, 180, 'add', False)]


def main(ref_root):
    sys.path[:0] = [os.path.join(ROOT, 'oracle', 'pyg_stub'), os.path.join(ref_root, 'graph-neural-operator')]
    import nn_conv            # the reference modules, unmodified
    import utilities
    C, kin = 6, 3
    rec = {}
    for i, (n_src, n_dst, E, aggr, rb) in enumerate(CASES):
        g = torch.Generator().manual_seed(120 + i)
        src = torch.randint(0, n_src - 3, (E,), generator=g)
        dst = torch.randint(2, n_dst, (E,), generator=g)
        ea = torch.randn(E, kin, generator=g)
        x_src = torch.randn(n_src, C, generator=g)
        x_dst = torch.randn(n_dst, C, generator=g)
        torch.manual_seed(2000 + i)
        conv = nn_conv.NNConv_old(C, C, utilities.DenseNet([kin, 16, 24, C * C], torch.nn.ReLU), aggr=aggr,
                                  root_weight=rb, bias=rb)
        union = torch.stack([src, n_src + dst])
        with torch.no_grad():
            out = conv(torch.cat([x_src, x_dst]), union, ea)[n_src:]
        pre = 'c%d_' % i
        rec[pre + 'case'] = np.array([n_src, n_dst, int(rb)])
        rec[pre + 'aggr'] = np.array(aggr)
        rec[pre + 'edge_index'] = torch.stack([src, dst]).numpy().astype(np.int64)
        rec[pre + 'edge_attr'] = ea.numpy()
        rec[pre + 'x_src'] = x_src.numpy()
        rec[pre + 'x_dst'] = x_dst.numpy()
        for k, v in conv.state_dict().items():
            rec[pre + 'sd_' + k] = v.numpy().copy()
        rec[pre + 'out'] = out.numpy()
    rec['n_cases'] = np.array(len(CASES))
    golden.save(os.path.join(ROOT, 'tests', 'golden', 'g12_bipartite_nnconv.npz'), **rec)
    print('wrote g12_bipartite_nnconv.npz: %d cases' % len(CASES))


if __name__ == '__main__':
    main(sys.argv[1])
