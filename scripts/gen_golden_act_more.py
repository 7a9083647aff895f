"""Write tests/golden/g14_edge_activations_more.npz by running the reference's own NNConv_old
(graph-neural-operator/nn_conv.py) and DenseNet (graph-neural-operator/utilities.py:201-227) classes, unmodified, over
oracle/pyg_stub on the CPU, with edge networks whose hidden activation is Hardtanh, ReLU6, Hardsigmoid, SELU, CELU,
Softsign or LogSigmoid:

    python scripts/gen_golden_act_more.py /path/to/graph-pde        # a checkout of neuraloperator/graph-pde

Cases: DenseNet([3, 16, 24, C * C], act) for each activation, at aggr add and mean.  Each case stores the module's
state dict after its seeded construction (the reference's init stream), its output and the gradients of
sum(out * g) with respect to x, edge_attr and every parameter, from the reference's own autograd.  The first layer's
weights are scaled by 4 so that the clamps saturate on a good share of the edges.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import golden  # noqa: E402

# (kind, parameter as the tests write it, module name, constructor arguments)
ACTS = [('relu6', 'None', 'ReLU6', ()), ('hardtanh', '-0.3,0.7', 'Hardtanh', (-0.3, 0.7)),
        ('hardsigmoid', 'None', 'Hardsigmoid', ()), ('selu', 'None', 'SELU', ()), ('celu', '0.5', 'CELU', (0.5,)),
        ('softsign', 'None', 'Softsign', ()), ('logsigmoid', 'None', 'LogSigmoid', ())]


def main(ref_root):
    sys.path[:0] = [os.path.join(ROOT, 'oracle', 'pyg_stub'), os.path.join(ref_root, 'graph-neural-operator')]
    import nn_conv            # the reference modules, unmodified
    import utilities
    g = torch.Generator().manual_seed(14)
    N, E, C, kin = 24, 160, 8, 3
    src = torch.randint(0, N - 3, (E,), generator=g)     # last 3 nodes: no out-edges
    dst = torch.randint(2, N, (E,), generator=g)         # first 2 nodes: no in-edges
    ei = torch.stack([src, dst])
    ea = torch.randn(E, kin, generator=g)
    x = torch.randn(N, C, generator=g)
    gout = torch.randn(N, C, generator=g)
    rec = dict(edge_index=ei.numpy().astype(np.int64), edge_attr=ea.numpy(), x=x.numpy(), grad_out=gout.numpy())
    cases = [(kind, p, name, args, aggr) for kind, p, name, args in ACTS for aggr in ('add', 'mean')]
    for i, (kind, p, name, args, aggr) in enumerate(cases):
        torch.manual_seed(1400 + i)
        nonlinearity = (lambda f, a: (lambda: f(*a)))(getattr(torch.nn, name), args)
        mlp = utilities.DenseNet([kin, 16, 24, C * C], nonlinearity)
        conv = nn_conv.NNConv_old(C, C, mlp, aggr=aggr)
        with torch.no_grad():
            mlp.layers[0].weight.mul_(4.0)
        pre = 'c%d_' % i
        rec[pre + 'case'] = np.array([kind, p, aggr])
        rec[pre + 'keys'] = np.array(list(conv.state_dict().keys()))
        for k, v in conv.state_dict().items():
            rec[pre + 'sd_' + k] = v.numpy().copy()
        xr = x.clone().requires_grad_()
        ear = ea.clone().requires_grad_()
        out = conv(xr, ei, ear)
        (out * gout).sum().backward()
        rec[pre + 'out'] = out.detach().numpy()
        rec[pre + 'grad_x'] = xr.grad.numpy()
        rec[pre + 'grad_edge_attr'] = ear.grad.numpy()
        for k, prm in conv.named_parameters():
            rec[pre + 'grad_' + k] = prm.grad.numpy().copy()
    rec['n_cases'] = np.array(len(cases))
    golden.save(os.path.join(ROOT, 'tests', 'golden', 'g14_edge_activations_more.npz'), **rec)
    print('wrote g14_edge_activations_more.npz: %d cases' % len(cases))


if __name__ == '__main__':
    main(sys.argv[1])
