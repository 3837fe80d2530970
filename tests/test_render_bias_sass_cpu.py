"""Where the render kernels' MLP epilogues read their bias from (no GPU needed: cuobjdump on the built library).

Fast mode copies both networks' bias blocks into shared memory once per CTA, so its epilogues issue no 64-bit global bias
load (`LDG.E.64.CONSTANT`, one per float2 of the thread's two columns).  The multi-frame kernels keep exactly those loads for
the per-frame rows of steps 0 and 3 (2 halves x 2 accumulator rows x 16 loads per step).  Exact mode has no shared memory
to spare and reads the bias from global memory: its kernels must still carry the loads, or the check would be vacuous.
"""
import os
import re
import shutil
import subprocess
from collections import Counter

import pytest

NVDIS = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@pytest.fixture(scope="module")
def bias_loads(built_lib):
    if not os.path.exists(NVDIS):
        pytest.skip("cuobjdump not found")
    sass = subprocess.run([NVDIS, "-sass", built_lib], capture_output=True, text=True, check=True).stdout
    loads, fn = Counter(), None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            k = re.search(r"render_kernelILb([01])ELb([01])ELb([01])E", m.group(1))
            f = re.search(r"render_frames_kernelILb([01])ELb([01])E", m.group(1))
            fn = ("single",) + tuple(int(x) for x in k.groups()) if k else ("frames",) + tuple(int(x) for x in f.groups()) if f else None
            if fn:
                loads[fn] += 0
            continue
        if fn and "LDG.E.64.CONSTANT" in line:
            loads[fn] += 1
    return loads


def test_fast_epilogues_read_the_bias_from_shared_memory(bias_loads):
    fast = [("single", 0, 0, 0), ("single", 0, 0, 1), ("single", 0, 1, 0)]
    assert all(k in bias_loads for k in fast), "render_kernel instantiations not found in the library"
    assert [bias_loads[k] for k in fast] == [0, 0, 0]
    assert bias_loads[("frames", 0, 0)] == bias_loads[("frames", 0, 1)] == 2 * 2 * 2 * 16


def test_exact_mode_reads_the_bias_from_global_memory(bias_loads):
    assert bias_loads[("single", 1, 0, 0)] > 0 and bias_loads[("single", 1, 1, 0)] > 0
