import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def oracle_factory():
    from oracle_api import new_oracle
    return new_oracle


@pytest.fixture(scope="session")
def cuda_lib():
    """The product library; GPU tests fail loudly (never skip to a fallback) when it is missing."""
    from openimucameracalibrator_b200 import calibrator
    return calibrator.load_library()


@pytest.fixture()
def gpu_factory(cuda_lib):
    from openimucameracalibrator_b200 import _capi as capi

    def make():
        return capi.CApi(cuda_lib, "icc_", 0)
    return make


@pytest.fixture(params=["sized", "tmem_always"])
def eval_path(request, monkeypatch):
    """Both Jacobian evaluation paths of launch_eval: the size-selected default (small problems: one warp per frame / cell) and the
    persistent shared-memory-parking kernel forced on (ICC_TMEM_ALWAYS), so that the small parity cases also pin the kernel BASELINE config 4 uses."""
    if request.param == "tmem_always":
        monkeypatch.setenv("ICC_TMEM_ALWAYS", "1")
    else:
        monkeypatch.delenv("ICC_TMEM_ALWAYS", raising=False)
    return request.param
