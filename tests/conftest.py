import os
import sys

import pytest

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
for p in (ROOT, TESTS):
    if p not in sys.path:
        sys.path.insert(0, p)

from cnmf_golden import load_golden  # noqa: E402  (tests/cnmf_golden.py; unique name: a foreign `tests` package exists in the image)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90)")


@pytest.fixture(scope="session", params=["sim_mu", "sim_cd", "sim_kl", "sim_nndsvd", "c1_mu", "c1_cd"])
def golden(request):
    return load_golden(request.param)
