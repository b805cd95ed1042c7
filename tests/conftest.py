import os
import sys

# tiny 3x3 numpy/LAPACK calls dominate the oracle; BLAS thread pools on many-core hosts make them pathologically slow
for _v in ('OMP_NUM_THREADS', 'OPENBLAS_NUM_THREADS', 'MKL_NUM_THREADS'):
    os.environ.setdefault(_v, '1')

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with `pytest -m gpu` on an H100)")
    config.addinivalue_line("markers", "reference: needs the reference tree (/root/reference or oracle/_ref)")


@pytest.fixture(scope='session')
def golden_dir():
    return GOLDEN
