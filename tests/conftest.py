import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on the H100 box)")


def pytest_collection_modifyitems(config, items):
    """Tests marked ``gpu`` are skipped (not failed) on a machine without a CUDA device: the product has no CPU path."""
    try:
        import torch
        have = torch.cuda.is_available()
    except Exception:
        have = False
    if have:
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (diffdock_b200 has no CPU fallback)")
    for it in items:
        if 'gpu' in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope='session')
def built_lib():
    import __graft_entry__ as g
    g.build()
    from diffdock_b200 import _lib
    return _lib.lib()
