"""The K-image training-step entries (NFB_TRAIN_IMAGES) without a GPU: declared, the ctypes mirrors laid out as the header's
structs, argument checks before any CUDA call, and the library's version."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "nfb.h")


@pytest.fixture(scope="module")
def capi(built_lib):
    from nerf import _capi
    return _capi


def _struct_fields(name):
    """(field name, array length) of `typedef struct { ... } name;` in include/nfb.h, in order."""
    body = re.search(r"typedef struct \{([^{}]*)\} " + name + ";", open(HEADER).read()).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    out = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            for part in decl.split(","):
                m = re.search(r"(\w+)\s*(?:\[(\d+)\])?\s*$", part.strip())
                out.append((m.group(1), int(m.group(2)) if m.group(2) else 1))
    return out


def test_header_declares_the_feature_at_version_131():
    h = open(HEADER).read()
    assert re.search(r"#define NFB_TRAIN_IMAGES 1\b", h)
    assert re.search(r"#define NFB_MAX_STEP_IMAGES 64\b", h)
    assert re.search(r"#define NFB_VERSION 131\b", h)
    for fn in ("nfb_sample_rays_images", "nfb_latent_rows_grad"):
        assert re.search(rf"\bint {fn}\(", h), fn


def test_version_is_131(capi):
    assert capi.lib.nfb_version() == 131
    assert capi.NFB_MAX_STEP_IMAGES == 64
    assert {"nfb_sample_rays_images", "nfb_latent_rows_grad"} <= set(capi.EXPORTS)


@pytest.mark.parametrize("name", ["NfbTrainImages", "NfbImageBatch"])
def test_ctypes_structs_match_the_header(capi, name):
    """Same fields in the same order; sizes and offsets as a C compiler lays out the header's types (LP64)."""
    st = getattr(capi, name)
    want = _struct_fields(name)
    assert [f for f, _ in st._fields_] == [f for f, _ in want]
    ctype_of = dict(st._fields_)
    for f, n in want:
        assert C.sizeof(ctype_of[f]) == n * (8 if f in ("maps", "poses", "expressions", "images", "background", "intrinsics") or
                                             name == "NfbImageBatch" else 4), f
    if name == "NfbTrainImages":
        assert [getattr(st, f).offset for f, _ in want] == [0, 8, 16, 24, 32, 40, 44, 48, 52, 56]
        assert C.sizeof(st) == 88
    else:
        assert [getattr(st, f).offset for f, _ in want] == [8 * i for i in range(11)]
        assert C.sizeof(st) == 88


def test_ray_map_mirror_layout(capi):
    """The sampler reads the device table of NfbRayMap through its own mirror (nfb_internal.h RayMapRec): 40 bytes, q_out at 24."""
    assert C.sizeof(capi.NfbRayMap) == 40 and capi.NfbRayMap.q_out.offset == 24 and capi.NfbRayMap.q_in.offset == 32


def _images(capi, n_images=2, H=8, W=8, background=True):
    buf = (C.c_float * 64)()
    d = capi.NfbTrainImages()
    d.maps = d.poses = d.expressions = d.images = C.addressof(buf)
    d.background = C.addressof(buf) if background else None
    d.n_images, d.height, d.width = n_images, H, W
    return d, buf


def test_sampler_argument_errors(capi):
    """Host-checkable misuse is refused before any CUDA call (a null handle is checked first, so these run without a device)."""
    lib = capi.lib
    d, keep = _images(capi)
    out = capi.NfbImageBatch()
    ptr = C.addressof(keep)
    assert lib.nfb_sample_rays_images(None, C.byref(d), ptr, 2, 16, ptr, 4, ptr, C.byref(out), None) == 1
    assert lib.nfb_sample_rays_images(None, None, ptr, 2, 16, ptr, 4, ptr, C.byref(out), None) == 1


def test_latent_rows_argument_errors(capi):
    lib = capi.lib
    buf = (C.c_float * 64)()
    p = C.addressof(buf)
    assert lib.nfb_latent_rows_grad(None, p, p, 1, p, 1, p, 0.0, None) == 1


def test_host_checks_in_the_source_order():
    """The checks the GPU-free tests cannot reach through a null handle are in nfb_api.cu ahead of the first CUDA call: K and n
    ranges, null tables, the background request, and the 64-image bound as NFB_ERR_UNSUPPORTED."""
    src = open(os.path.join(ROOT, "4d-facial-avatars_b200", "csrc", "nfb_api.cu")).read()
    body = src[src.index("int nfb_sample_rays_images("):]
    body = body[:body.index("\n}\n")]
    first_cuda = body.index("cudaSetDevice")
    for check in ("K < 1", "n < 1", "n > nfb::kSmpMax", "max_rounds < 1", "K > NFB_MAX_STEP_IMAGES", "!d->maps", "!d->images",
                  "out->background && !d->background", "< n)"):
        assert 0 <= body.find(check) < first_cuda, check
    assert "return NFB_ERR_UNSUPPORTED" in body[:first_cuda]
    body = src[src.index("int nfb_latent_rows_grad("):]
    body = body[:body.index("\n}\n")]
    for check in ("K < 1", "n_rows < 1", "!table_grads", "K > NFB_MAX_STEP_IMAGES"):
        assert 0 <= body.find(check) < body.index("cudaSetDevice"), check


def test_python_surface_raises_for_sharded_steps(built_lib):
    """world > 1 is not implemented for K-image steps; the check comes before any device work."""
    from nerf import fused_train
    tr = fused_train.FusedTrainer.__new__(fused_train.FusedTrainer)

    class Data:
        H = W = 8
        n_images = 2
    with pytest.raises(NotImplementedError):
        tr._check_images(Data(), 2, 16, world=2)
    with pytest.raises(ValueError):
        fused_train.FusedTrainer._check_images(tr, Data(), 65, 16, world=1)
