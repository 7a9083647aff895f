import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason='no CUDA device in this container')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope='session')
def golden_dir():
    return GOLDEN


@pytest.fixture(params=['auto', 'off'])
def edge_kernel_mode(request):
    """Run a GPU test under both application paths: 'auto' (small / low out-degree graphs use per-edge kernel matrices,
    formulation B) and 'off' (always the persistent fused kernel, formulation C) -- most test graphs are small enough
    for 'auto' to pick B, and both paths must meet the same tolerances."""
    from graph_pde_b200 import nn_conv
    old = nn_conv._EDGE_KERNELS
    nn_conv._EDGE_KERNELS = request.param
    yield request.param
    nn_conv._EDGE_KERNELS = old
