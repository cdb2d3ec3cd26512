import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def oracle():
    from tests.orc import Oracle, build_oracle
    build_oracle(with_ref=True)
    return Oracle()


@pytest.fixture(scope="session")
def refs():
    from tests.orc import Ref
    if not Ref.available():
        pytest.skip("oracle/_ref not built (needs /root/reference)")
    return {k: Ref(k) for k in ("f32s", "f32f", "q28")}
