"""What the compiler made of the render kernel's MLP epilogues (no GPU needed: cuobjdump on the built library).

The fast-mode evaluation kernel (`render_kernel<false, false, false>`, the headline) issues no global store between an MLP
batch's last HGMMA and the next WARPGROUP.ARRIVE, i.e. in the epilogues that run between two steps' MMAs: the activation
probe's dumps live only in the probe instantiation (`render_kernel<false, false, true>`), which must have them, or the check
would pass vacuously.  Exact mode's steps are a runtime loop, whose epilogue does not sit between two MMA batches in the
code; there the production kernel must simply carry fewer global stores than the probe one.  The training forward
(`<EXACT, true, false>`) stores its activation records from the same epilogues by design and has no probe instantiation.
"""
import os
import re
import shutil
import subprocess
from collections import defaultdict

import pytest

NVDIS = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


def epilogue_stores(lib):
    """Per render_kernel instantiation (EXACT, SAVE, PROBE): [global stores between each HGMMA and the next
    WARPGROUP.ARRIVE], and the global stores of the whole kernel."""
    sass = subprocess.run([NVDIS, "-sass", lib], capture_output=True, text=True, check=True).stdout
    res, total = defaultdict(list), defaultdict(int)
    fn = None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            k = re.search(r"render_kernelILb([01])ELb([01])ELb([01])E", m.group(1))
            fn = tuple(int(x) for x in k.groups()) if k else None
            after_mma, n = False, 0
            continue
        if fn is None or not re.match(r"\s+/\*[0-9a-f]{4,}\*/", line):
            continue
        if re.search(r"\bSTG\b", line):
            total[fn] += 1
        if "HGMMA" in line:
            after_mma, n = True, 0
        elif "WARPGROUP.ARRIVE" in line:
            if after_mma:
                res[fn].append(n)
            after_mma = False
        elif after_mma and re.search(r"\bSTG\b", line):
            n += 1
    return res, total


@pytest.fixture(scope="module")
def stores(built_lib):
    if not os.path.exists(NVDIS):
        pytest.skip("cuobjdump not found")
    return epilogue_stores(built_lib)


def test_no_global_store_in_the_fast_epilogues(stores):
    epi, _ = stores
    prod, probe = epi[(0, 0, 0)], epi[(0, 0, 1)]
    assert prod and probe, "render_kernel instantiations not found in the library"
    assert sum(prod) == 0, prod
    assert sum(probe) > 0, "the probe instantiation has no epilogue stores: the check would be vacuous"


def test_exact_mode_probe_code_only_in_the_probe_kernel(stores):
    _, total = stores
    assert 0 < total[(1, 0, 0)] < total[(1, 0, 1)]


def test_training_forward_has_no_probe_instantiation(stores):
    _, total = stores
    assert (0, 1, 1) not in total and (1, 1, 1) not in total
    assert (0, 1, 0) in total and (1, 1, 0) in total
