import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on the GPU box)")


@pytest.fixture(scope="session")
def orc():
    import oracle
    oracle.build()
    return oracle


@pytest.fixture(scope="session")
def gpu_ctx():
    import oramacore_b200 as ob
    ctx = ob.Context(0)  # raises loudly when the CUDA extension / device is missing
    yield ctx
    ctx.close()
