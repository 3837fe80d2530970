"""C-ABI checks that need no GPU: the library builds, loads, and exports every symbol include/nfb.h declares;
host-only helpers behave."""
import ctypes
import os
import re

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_exports_match_header(built_lib):
    header = open(os.path.join(ROOT, "include", "nfb.h")).read()
    declared = set(re.findall(r"^(?:int|const char\*)\s+(nfb_\w+)\s*\(", header, flags=re.M))
    assert {"nfb_create", "nfb_render_forward", "nfb_set_frame", "nfb_load_weights"} <= declared
    lib = ctypes.CDLL(built_lib)
    missing = [name for name in declared if not hasattr(lib, name)]
    assert not missing, missing
    lib.nfb_version.restype = ctypes.c_int
    assert lib.nfb_version() >= 100
    lib.nfb_strerror.restype = ctypes.c_char_p
    assert lib.nfb_strerror(0) == b"ok" and b"sm_90a" in lib.nfb_strerror(2)


def test_host_linspace_scalar_formula(built_lib):
    lib = ctypes.CDLL(built_lib)
    for n in (2, 3, 64, 128, 257):
        buf = (ctypes.c_float * n)()
        assert lib.nfb_host_linspace(buf, n) == 0
        got = torch.tensor(list(buf))
        ref = torch.linspace(0.0, 1.0, n)
        assert got[0] == 0.0 and got[-1] == 1.0
        assert float((got - ref).abs().max()) <= 1.2e-7  # ATen's vectorised halves may differ by 1 ulp
    assert lib.nfb_host_linspace(None, 4) != 0


def test_invalid_arguments_return_codes(built_lib):
    lib = ctypes.CDLL(built_lib)
    assert lib.nfb_create(None, 0, None) == 1            # NFB_ERR_INVALID, before any CUDA call
    assert lib.nfb_destroy(None) == 1
    assert lib.nfb_launch_count(None, None) == 1


def test_adam_dev_struct_matches_the_header(built_lib, tmp_path):
    """_capi.NfbAdamDev has the size and field offsets a C compiler gives include/nfb.h's NfbAdamDev (the schedule's constants
    are double since version 131; a float mirror would hand the device shifted fields)."""
    import shutil
    import subprocess
    from nerf import _capi
    cc = shutil.which("cc") or shutil.which("gcc")
    assert cc, "a C compiler is needed to read the header's layout"
    fields = [name for name, _ in _capi.NfbAdamDev._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "nfb.h"\nint main(void) {\n'
                   '  printf("%zu\\n", sizeof(NfbAdamDev));\n'
                   + "".join(f'  printf("%zu\\n", offsetof(NfbAdamDev, {f}));\n' for f in fields) + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    want = [ctypes.sizeof(_capi.NfbAdamDev)] + [getattr(_capi.NfbAdamDev, f).offset for f in fields]
    assert got == want, dict(zip(["sizeof"] + fields, zip(got, want)))
    assert {f: t for f, t in _capi.NfbAdamDev._fields_ if f in ("lr0", "decay_factor", "decay_steps")} == dict.fromkeys(
        ("lr0", "decay_factor", "decay_steps"), ctypes.c_double)


def test_buffer_epoch_is_exported_and_rejects_null(built_lib):
    lib = ctypes.CDLL(built_lib)
    out = ctypes.c_longlong(-5)
    assert lib.nfb_buffer_epoch(None, ctypes.byref(out)) == 1 and out.value == -5  # NFB_ERR_INVALID, nothing written
    assert lib.nfb_buffer_epoch(None, None) == 1


def test_python_surface_matches_reference_names(built_lib):
    import nerf
    for name in ["load_flame_data", "CfgNode", "get_embedding_function", "get_ray_bundle", "img2mse", "load_llff_data",
                 "meshgrid_xy", "models", "mse2psnr", "run_one_iter_of_nerf", "dump_rays", "GaussianSmoothing",
                 "predict_and_render_radiance"]:
        assert hasattr(nerf, name), name
    m = nerf.models.ConditionalBlendshapePaperNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4,
                                                        include_input_xyz=True, include_input_dir=False)
    import nerface_oracle as O
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == O.PAPER_MODEL_SHAPES
    x = torch.randn(5, 87)
    p = {k: v.detach() for k, v in m.state_dict().items()}
    e, l = torch.randn(76), torch.randn(32)
    assert torch.allclose(m(x, e, l), O.mlp_forward(p, x, e, l), atol=1e-6)


def test_render_requires_cuda(built_lib):
    import nerf
    import pytest
    m = nerf.models.ConditionalBlendshapePaperNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4,
                                                        include_input_xyz=True, include_input_dir=False)
    cfg = nerf.CfgNode(dict(nerf=dict(use_viewdirs=True, validation=dict(num_coarse=8, num_fine=0, perturb=False, lindisp=False,
                       radiance_field_noise_std=0.0, white_background=False, chunksize=64)), dataset=dict(no_ndc=True, near=0.2, far=0.8)))
    ro = torch.zeros(4, 4, 3)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        nerf.run_one_iter_of_nerf(4, 4, 1.0, m, None, ro, ro + 1, cfg, mode="validation", expressions=torch.zeros(76),
                                  latent_code=torch.zeros(32))
