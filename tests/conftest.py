import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def pytest_collection_modifyitems(config, items):
    """GPU tests fail loudly (not skip) on a box that has a GPU but cannot load the native library;
    on a box without a GPU they are deselected by `-m "not gpu"`."""
    return
