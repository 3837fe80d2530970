"""Exact-grad mode's C ABI without a GPU: the header declares NFB_PREC_EXACT_GRAD and its feature macro, the Python binding mirrors
the structs it extends, and the Python surface accepts the mode's name."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header():
    with open(os.path.join(ROOT, "include", "nfb.h")) as f:
        return f.read()


def test_header_declares_the_mode():
    h = header()
    assert re.search(r"enum \{ NFB_PREC_FAST = 0, NFB_PREC_EXACT = 1, NFB_PREC_EXACT_GRAD = 2 \};", h)
    assert "#define NFB_EXACT_GRAD 1" in h
    assert "#define NFB_VERSION 131" in h  # the feature is announced by its macro, as NFB_REPRODUCIBLE_BACKWARD was


def _layout(tmp_path, struct, fields):
    cc = shutil.which("cc") or shutil.which("gcc")
    assert cc, "a C compiler is needed to read the header's layout"
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nfb.h"\nint main(void) {\n'
                   f'  printf("%zu\\n", sizeof({struct}));\n  printf("%d\\n", (int)NFB_PREC_EXACT_GRAD);\n'
                   + "".join(f'  printf("%zu\\n", offsetof({struct}, {f}));\n' for f in fields) + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    return [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]


@pytest.mark.parametrize("struct", ["NfbWeightDebug", "NfbTrainDebug", "NfbSampling"])
def test_ctypes_structs_match_the_header(built_lib, tmp_path, struct):
    from nerf import _capi
    cls = getattr(_capi, struct)
    fields = [name for name, _ in cls._fields_]
    got = _layout(tmp_path, struct, fields)
    want = [ctypes.sizeof(cls), _capi.NFB_PREC_EXACT_GRAD] + [getattr(cls, f).offset for f in fields]
    assert got == want, dict(zip(["sizeof", "NFB_PREC_EXACT_GRAD"] + fields, zip(got, want)))
    if struct == "NfbWeightDebug":
        assert fields[-2:] == ["bwd_lo", "bwd_lo_bytes"]


def test_python_accepts_exact_grad(built_lib):
    from nerf import _capi, _engine
    before = _engine.get_precision()
    try:
        _engine.set_precision("exact_grad")
        assert _engine.get_precision() == "exact_grad"
        assert _engine.PRECISIONS == {"fast": 0, "exact": 1, "exact_grad": 2}
        assert _engine.PRECISIONS["exact_grad"] == _capi.NFB_PREC_EXACT_GRAD
        with pytest.raises(ValueError):
            _engine.set_precision("exact_grads")
    finally:
        _engine.set_precision(before)


def test_library_is_built_with_the_mode(built_lib):
    """The exact-grad instantiations are in the library (the no-FP-atomic scan of test_reproducible_cpu.py covers them)."""
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not found")
    names = subprocess.run([tool, "-elf", built_lib], capture_output=True, text=True, check=True).stdout
    for k in ("render_hilo_kernel", "chain_x3_kernel", "dw_x3_kernel", "row_x3_kernel", "raysum_x3_kernel", "bwd_lo_kernel"):
        assert k in names, k
