"""Write tests/golden/g10_edge_activations.npz by running the reference's own NNConv_old
(graph-neural-operator/nn_conv.py) and DenseNet (graph-neural-operator/utilities.py:201-227) classes, unmodified, over
oracle/pyg_stub on the CPU, with edge networks whose hidden activation is not ReLU:

    python scripts/gen_golden_act.py /path/to/graph-pde        # a checkout of neuraloperator/graph-pde

Cases: DenseNet([3, 16, 24, C * C], act) for LeakyReLU(0.1), ELU(0.7), Tanh and Sigmoid, each at aggr add and mean.
Each case stores the module's state dict after its seeded construction (the reference's init stream) and its output.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import golden  # noqa: E402

# (kind, parameter, module factory name, constructor arguments)
ACTS = [('leaky_relu', 0.1, 'LeakyReLU', (0.1,)), ('elu', 0.7, 'ELU', (0.7,)), ('tanh', 0.0, 'Tanh', ()),
        ('sigmoid', 0.0, 'Sigmoid', ())]


def main(ref_root):
    sys.path[:0] = [os.path.join(ROOT, 'oracle', 'pyg_stub'), os.path.join(ref_root, 'graph-neural-operator')]
    import nn_conv            # the reference modules, unmodified
    import utilities
    g = torch.Generator().manual_seed(10)
    N, E, C, kin = 24, 160, 8, 3
    src = torch.randint(0, N - 3, (E,), generator=g)     # last 3 nodes: no out-edges
    dst = torch.randint(2, N, (E,), generator=g)         # first 2 nodes: no in-edges
    ei = torch.stack([src, dst])
    ea = torch.randn(E, kin, generator=g)
    x = torch.randn(N, C, generator=g)
    rec = dict(edge_index=ei.numpy().astype(np.int64), edge_attr=ea.numpy(), x=x.numpy())
    cases = []
    for kind, p, name, args in ACTS:
        for aggr in ('add', 'mean'):
            cases.append((kind, p, name, args, aggr))
    for i, (kind, p, name, args, aggr) in enumerate(cases):
        torch.manual_seed(1000 + i)
        nonlinearity = (lambda f, a: (lambda: f(*a)))(getattr(torch.nn, name), args)
        mlp = utilities.DenseNet([kin, 16, 24, C * C], nonlinearity)
        conv = nn_conv.NNConv_old(C, C, mlp, aggr=aggr)
        with torch.no_grad():
            out = conv(x, ei, ea)
        pre = 'c%d_' % i
        rec[pre + 'case'] = np.array([kind, str(p), aggr])
        rec[pre + 'keys'] = np.array(list(conv.state_dict().keys()))
        for k, v in conv.state_dict().items():
            rec[pre + 'sd_' + k] = v.numpy().copy()
        rec[pre + 'out'] = out.numpy()
    rec['n_cases'] = np.array(len(cases))
    golden.save(os.path.join(ROOT, 'tests', 'golden', 'g10_edge_activations.npz'), **rec)
    print('wrote g10_edge_activations.npz: %d cases' % len(cases))


if __name__ == '__main__':
    main(sys.argv[1])
