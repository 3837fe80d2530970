import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "oracle"), os.path.join(ROOT, "4d-facial-avatars_b200"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def built_lib():
    import __graft_entry__ as ge
    ge.build()
    return os.path.join(ROOT, "4d-facial-avatars_b200", "lib", "libnfb.so")
