"""The input-gradient entry point of the C ABI is exported and the header version says so (no GPU needed)."""
import ctypes
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib(built_lib):
    return ctypes.CDLL(built_lib)


def test_backward_ex_exported_at_version_131(lib):
    lib.nfb_version.restype = ctypes.c_int
    assert lib.nfb_version() == 131
    assert hasattr(lib, "nfb_render_backward_ex")
    with open(os.path.join(ROOT, "include", "nfb.h")) as f:
        h = f.read()
    assert "#define NFB_VERSION 131" in h and "NfbInputGrads" in h


def test_backward_ex_rejects_null_handle(lib):
    lib.nfb_render_backward_ex.restype = ctypes.c_int
    lib.nfb_render_backward_ex.argtypes = [ctypes.c_void_p] * 9
    assert lib.nfb_render_backward_ex(None, None, None, None, None, None, None, None, None) == 1  # NFB_ERR_INVALID
