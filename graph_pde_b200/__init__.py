"""graph_pde_b200 -- H100-native (sm_90a) implementation of the NNConv hot path of
neuraloperator/graph-pde: the edge-conditioned convolution iterated inside KernelNN and the MGKN
V-cycle.  Public surface mirrors the reference's operator API:

    from graph_pde_b200.nn_conv import NNConv_old, NNConv      # reference: nn_conv.py / torch_geometric.nn
    from graph_pde_b200.gauss import GaussianNNConv           # reference: nn_conv.py NNConv_Gaussian
    from graph_pde_b200.models import KernelNN, KernelInduced, MKGN, MGKN

(the directory is also reachable as ``graph-pde_b200`` through a symlink; Python cannot import a
hyphenated name).
"""
from . import _lib  # noqa: F401
from .nn_conv import NNConv, NNConv_old, ECConv, stats, clear_caches  # noqa: F401
from .gcn import GCNConv  # noqa: F401
from .gauss import GaussianNNConv  # noqa: F401

__version__ = '0.1.0'
from .capture import GraphedForward, GraphedTrainStep  # noqa: F401,E402
