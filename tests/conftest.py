import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def oracle_api():
    from oracle import oracle
    return oracle.api()


@pytest.fixture(scope="session")
def gpu_api():
    """The product library bound to cuda:0.  GPU tests fail (not skip) when it is missing: a silent
    fallback would void every parity claim."""
    import torch
    assert torch.cuda.is_available(), "gpu-marked test run without a CUDA device"
    from snappydata_b200 import capi
    api = capi.product_api()
    api.check(api.init(0))
    return api
