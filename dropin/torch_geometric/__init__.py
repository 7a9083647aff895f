"""Minimal stand-in for the parts of torch_geometric the reference scripts import, with NNConv backed by the
H100 library.  Put the parent directory first on sys.path:

    from torch_geometric.nn import NNConv            (MGKN_general_darcy2d.py:8)
    from torch_geometric.data import Data, DataLoader (UAI1_full_resolution.py:6)

It is NOT PyG: only NNConv / Data / DataLoader (with block-diagonal batching) exist.
"""
__version__ = '0.0-graph-pde-b200-shim'
