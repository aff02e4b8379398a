import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with -m gpu)")


GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="session")
def golden():
    import numpy as np
    import torch

    def load(name):
        with np.load(os.path.join(GOLDEN, name + ".npz")) as z:
            return {k: torch.from_numpy(z[k]) for k in z.files}

    return load
