"""The multi-frame entries (NFB_MULTI_FRAME) without a GPU: declared, exported, argument checks before any CUDA call, and what
the compiler made of the multi-frame render kernel's epilogues."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVDIS = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@pytest.fixture(scope="module")
def capi(built_lib):
    from nerf import _capi
    return _capi


def test_header_declares_the_feature():
    h = open(os.path.join(ROOT, "include", "nfb.h")).read()
    assert re.search(r"#define NFB_MULTI_FRAME 1", h)
    assert re.search(r"#define NFB_MAX_FRAMES 1024", h)
    for fn in ("nfb_set_frames", "nfb_render_forward_frames", "nfb_render_forward_frames_train", "nfb_render_backward_frames"):
        assert re.search(rf"\bint {fn}\(", h), fn


def test_null_handles_and_arguments_are_invalid(capi):
    lib = capi.lib
    buf = (C.c_float * 256)()
    assert lib.nfb_set_frames(None, buf, buf, 1, None) == 1
    assert lib.nfb_render_forward_frames(None, None, None, None, None, None, None) == 1
    assert lib.nfb_render_forward_frames_train(None, None, None, None, None, None, None) == 1
    assert lib.nfb_render_backward_frames(None, None, None, None, None, None, None, None, None, None) == 1


def frames_epilogue_stores(lib):
    """[global stores between each HGMMA and the next WARPGROUP.ARRIVE] of render_frames_kernel<false, false>."""
    sass = subprocess.run([NVDIS, "-sass", lib], capture_output=True, text=True, check=True).stdout
    res, fn, after_mma, n = [], False, False, 0
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = "render_frames_kernelILb0ELb0E" in m.group(1)
            after_mma, n = False, 0
            continue
        if not fn or not re.match(r"\s+/\*[0-9a-f]{4,}\*/", line):
            continue
        if "HGMMA" in line:
            after_mma, n = True, 0
        elif "WARPGROUP.ARRIVE" in line:
            if after_mma:
                res.append(n)
            after_mma = False
        elif after_mma and re.search(r"\bSTG\b", line):
            n += 1
    return res


def test_no_global_store_in_the_multi_frame_fast_epilogues(built_lib):
    if not os.path.exists(NVDIS):
        pytest.skip("cuobjdump not found")
    epi = frames_epilogue_stores(built_lib)
    assert epi, "render_frames_kernel<false, false> not found in the library"
    assert sum(epi) == 0, epi


def test_train_debug_struct_matches_header_appended_fields(capi):
    """nerf._capi.NfbTrainDebug declares the fields of include/nfb.h's NfbTrainDebug, in the header's order, at offsets that
    only grow: a field appended to one but not the other, or two swapped, reads the wrong device pointer.  The last eleven
    fields are the six multi-frame ones, followed by the five parameter-gradient ones appended after them."""
    h = open(os.path.join(ROOT, "include", "nfb.h")).read()
    body = re.search(r"typedef struct \{([^{}]*)\} NfbTrainDebug;", h).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        for part in decl.split(","):
            m = re.search(r"(\w+)\s*(\[\d+\])?\s*$", part.strip())
            names.append(m.group(1))
    fields = [f[0] for f in capi.NfbTrainDebug._fields_]
    assert fields == names
    offsets = [getattr(capi.NfbTrainDebug, f).offset for f in fields]
    assert offsets == sorted(offsets) and len(set(offsets)) == len(offsets)
    assert fields[-11:] == ["n_frames", "frame", "frame_table", "frame_cond", "ray_sums", "frame_sums", "dw_partials",
                            "dw_slot_floats", "dw_parts", "dw_pe_only", "ray_bias_sums"]
    assert C.sizeof(dict(capi.NfbTrainDebug._fields_)["frame_table"]) == 2 * C.sizeof(C.c_void_p)
    assert C.sizeof(dict(capi.NfbTrainDebug._fields_)["dw_parts"]) == 2 * C.sizeof(C.c_int32)