"""Drop-in for graph-neural-operator/nn_conv.py: put this directory FIRST on sys.path (or PYTHONPATH) and the
reference scripts' ``from nn_conv import NNConv_old`` (UAI1_full_resolution.py:9) resolves to this library's op.
Whole-module checkpoints pickled by the reference bind to the class path ``nn_conv.NNConv_old`` -- kept."""
import os
import sys

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)

from graph_pde_b200.nn_conv import NNConv_old as _Base  # noqa: E402
from graph_pde_b200.nn_conv import NNConv as _UpstreamNNConv  # noqa: E402


class NNConv_old(_Base):
    pass


# The reference's nn_conv.py also defines `NNConv` (a diagonal-kernel variant, nn_conv.py:8-96) and
# `NNConv_Gaussian`; neither is instantiated by any script (SURVEY section 2), so they are not provided.
NNConv_old.__module__ = 'nn_conv'
ECConv = _UpstreamNNConv
