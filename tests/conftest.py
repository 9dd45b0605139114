import os
import sys

import pytest

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (_ROOT, os.path.join(_ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


@pytest.fixture(scope="session")
def built():
    from immesh_b200 import build
    build.build_oracle()
    build.build_emu()
    return True


@pytest.fixture(scope="session")
def emu_lib(built):
    from immesh_b200 import api, build
    return api.load_library(build.EMU)


@pytest.fixture(scope="session")
def cuda_lib():
    from immesh_b200 import api
    return api.load_library()  # fails loudly if the CUDA extension is missing
