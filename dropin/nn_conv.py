"""Drop-in for graph-neural-operator/nn_conv.py: put this directory FIRST on sys.path (or PYTHONPATH) and the
reference scripts' ``from nn_conv import NNConv_old`` (UAI1_full_resolution.py:9) and ``from nn_conv import NNConv,
NNConv_old`` (neurips1_GKN.py:10, neurips5_GKN.py:10) resolve to this library's ops, and so does the module's third
class, ``NNConv_Gaussian``.  Whole-module checkpoints pickled by the reference bind to the class paths
``nn_conv.NNConv_old``, ``nn_conv.NNConv`` and ``nn_conv.NNConv_Gaussian`` -- kept."""
import os
import sys

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)

from graph_pde_b200.nn_conv import NNConv_old as _Base  # noqa: E402
from graph_pde_b200.nn_conv import NNConv as _UpstreamNNConv  # noqa: E402
from graph_pde_b200.nn_conv import DiagNNConv as _Diag  # noqa: E402
from graph_pde_b200.gauss import GaussianNNConv as _Gauss  # noqa: E402


class NNConv_old(_Base):
    pass


class NNConv(_Diag):
    """The reference's diagonal-kernel conv (nn_conv.py:8-96), imported by neurips1_GKN.py / neurips5_GKN.py."""
    pass


class NNConv_Gaussian(_Gauss):
    """The reference's Gaussian-kernel conv (nn_conv.py:99-194)."""
    pass


# The reference's ECConv (nn_conv.py:288) names the diagonal class; here ECConv stays the upstream torch_geometric
# NNConv (INTEGRATION 1).
NNConv_old.__module__ = 'nn_conv'
NNConv.__module__ = 'nn_conv'
NNConv.__qualname__ = 'NNConv'
NNConv_Gaussian.__module__ = 'nn_conv'
ECConv = _UpstreamNNConv
