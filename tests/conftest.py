import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


@pytest.fixture(scope="session")
def oracle():
    """The plain-C restatement (oracle/liboracle.so); compiled on demand (gcc is in the image on both boxes)."""
    from oracle import oracle as om
    if not os.path.exists(om.Oracle.path):
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-s", "liboracle.so"], check=True)
    return om.Oracle()


@pytest.fixture(scope="session")
def reference():
    """The unmodified reference compiled in place (oracle/_ref/libcpi_ref.so); prebuilt, may be absent."""
    from oracle import oracle as om
    if not om.Reference.available():
        pytest.skip("oracle/_ref/libcpi_ref.so not built (needs the rpng/cpi checkout at CPI_REFERENCE, by default /root/reference)")
    return om.Reference()


@pytest.fixture(scope="session")
def golden():
    import numpy as np
    g = os.path.join(ROOT, "tests", "golden")
    return dict(preint=np.load(os.path.join(g, "preint_golden.npz")), factor=np.load(os.path.join(g, "factor_golden.npz")))


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from cpi_b200 import capi
    capi.load()      # raises loudly if the extension was not built
    return torch
