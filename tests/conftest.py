import os
import sys

import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')
    # The CPU oracles / reference modules evaluated inside the tests get at most 32 OpenMP threads.  On many-core GPU hosts
    # PyTorch's default (every hardware thread) can be far slower than 32 threads for the same frame, above all on a loaded
    # host (bench.py calibrates its CPU arm the same way).
    n = str(min(32, os.cpu_count() or 1))
    os.environ.setdefault('OMP_NUM_THREADS', n)
    os.environ.setdefault('MKL_NUM_THREADS', n)
    import torch
    torch.set_num_threads(int(n))


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)
