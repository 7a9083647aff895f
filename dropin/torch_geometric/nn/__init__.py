import os
import sys

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)

from graph_pde_b200.gcn import GCNConv  # noqa: E402,F401
from graph_pde_b200.nn_conv import NNConv  # noqa: E402,F401
