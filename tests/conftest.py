import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: run with -m gpu)")
    # The compiled reference (oracle/_ref) DEFines the detectron2:: op schemas; load it before detectron2_b200.ops
    # so that our library only adds CUDA kernels next to the reference's CPU ones (see ops.register_detectron2_namespace).
    try:
        from oracle import oracle as orc

        orc.load_reference()
    except Exception:
        pass


@pytest.fixture(scope="session")
def golden():
    import numpy as np

    def load(name):
        return np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))

    return load
