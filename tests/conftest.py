import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')
    # the shared libraries are build artefacts (git-ignored): build them once if a fresh
    # checkout runs the tests before __graft_entry__.build() (nvcc cross-compiles without a GPU)
    lib = os.path.join(ROOT, 'neurite_b200', 'lib', 'libneurite_b200.so')
    ora = os.path.join(ROOT, 'oracle', 'c', 'liboracle.so')
    if not (os.path.exists(lib) and os.path.exists(ora)):
        import subprocess
        subprocess.check_call([sys.executable, os.path.join(ROOT, '__graft_entry__.py')])


def golden_names(prefix):
    return sorted(f[:-4] for f in os.listdir(GOLDEN) if f.startswith(prefix) and f.endswith('.npz'))


def load_golden(name):
    import numpy as np
    return np.load(os.path.join(GOLDEN, name + '.npz'), allow_pickle=False)


@pytest.fixture(scope='session')
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    return torch.device('cuda:0')
