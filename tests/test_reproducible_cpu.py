"""Guard for the bit-reproducible backward (include/nfb.h): no floating-point atomic addition anywhere in the library.  The
order in which atomics land changes from run to run, so one float atomicAdd or red.*.f32 makes gradients differ in their last
bits between identical calls.  The only atomic additions allowed are the integer cycle counters of the NFB_TIMERS phase
timers; max / min atomics do not depend on order and are not checked."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "4d-facial-avatars_b200", "csrc")


def _sources():
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".cuh", ".h")):
            yield name, open(os.path.join(CSRC, name)).read()


def _code(text):
    """The source without comments (a comment may name what the code no longer does)."""
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return re.sub(r"//[^\n]*", "", text)


def test_no_float_atomic_add_in_sources():
    bad = []
    for name, text in _sources():
        code = _code(text)
        for m in re.finditer(r"\b(?:unsafeAtomicAdd|atomicAdd(?:_block|_system)?)\s*\(", code):
            line = code[m.start():code.find("\n", m.start())]
            if "(unsigned long long)" not in line:  # the NFB_TIMERS counters: integer cycles
                bad.append((name, line.strip()))
        for m in re.finditer(r"\b(?:red|atom)(?:\.\w+)*\.(?:f16x2|bf16x2|f16|bf16|f32|f64)\b", code):
            bad.append((name, m.group(0)))
    assert not bad, bad


def test_timer_counters_are_the_only_atomic_add():
    allowed = [(name, line) for name, text in _sources() for line in _code(text).splitlines() if "atomicAdd" in line]
    assert all(name == "nfb_render_common.cuh" and "(unsigned long long)" in line for name, line in allowed), allowed


def test_no_float_atomic_add_in_the_built_library(built_lib):
    """What the compiler emitted, not just what the sources say: no RED / ATOM instruction that adds floating-point values."""
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not found")
    sass = subprocess.run([tool, "-sass", built_lib], capture_output=True, text=True, check=True).stdout
    assert "Function :" in sass
    found = sorted(set(re.findall(r"\b(?:RED|ATOM)\w*\.E\.ADD\.(?:F16\w*|BF16\w*|F32|F64)[\w.]*", sass)))
    assert not found, found
