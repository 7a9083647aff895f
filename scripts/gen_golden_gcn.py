"""Write tests/golden/g9_gcn_net.npz by running the reference's own GCN_Net class, taken by `ast` from
multipole-graph-neural-operator/neurips4_GCN.py unmodified, over the fp64 GCNConv restatement of tests/gcn_oracle.py
on the CPU:

    python scripts/gen_golden_gcn.py /path/to/graph-pde        # a checkout of neuraloperator/graph-pde

One 6 x 5 lattice of the reference's grid_edge order, width 32, ker_width 16, depth 2.  The record holds the edge_index,
the input, the state dict after the seeded construction (the reference's init stream) and the fp64 output.
"""
import ast
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import golden  # noqa: E402
from tests import gcn_oracle  # noqa: E402
from graph_pde_b200.graphs import grid_edge  # noqa: E402


def reference_class(path, name):
    src = open(path).read()
    node = next(n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == name)
    ns = {'torch': torch, 'F': F, 'nn': torch.nn, 'GCNConv': gcn_oracle.GCNConv}
    exec(compile(ast.Module(body=[node], type_ignores=[]), path, 'exec'), ns)
    return ns[name]


def main(ref_root):
    GCN_Net = reference_class(os.path.join(ref_root, 'multipole-graph-neural-operator', 'neurips4_GCN.py'), 'GCN_Net')
    _, ei = grid_edge(6, 5)
    g = torch.Generator().manual_seed(9)
    x = torch.randn(ei.max().item() + 1, 1, generator=g, dtype=torch.float64)
    torch.manual_seed(90)
    net = GCN_Net(32, 16, 2, in_width=1).double()

    class Data(object):
        pass
    d = Data()
    d.x, d.edge_index = x, ei
    with torch.no_grad():
        out = net(d)
    rec = dict(edge_index=ei.numpy(), x=x.numpy(), out=out.numpy(), keys=np.array(list(net.state_dict().keys())))
    for k, v in net.state_dict().items():
        rec['sd_' + k] = v.numpy().copy()
    golden.save(os.path.join(ROOT, 'tests', 'golden', 'g9_gcn_net.npz'), **rec)
    print('wrote g9_gcn_net.npz: %d nodes, %d edges' % (x.size(0), ei.size(1)))


if __name__ == '__main__':
    main(sys.argv[1])
