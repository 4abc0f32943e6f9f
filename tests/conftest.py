import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100; everything else runs on CPU")


@pytest.fixture(scope="session")
def engine():
    """The cached libb200gs handle on cuda:0 -- fails loudly if the CUDA library or GPU is missing."""
    from spark_sklearn_b200.estimators import get_engine
    return get_engine(0)


def golden(name):
    import numpy as np
    return np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"), allow_pickle=False)
