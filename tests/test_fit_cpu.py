"""Fitting steps over several images (NFB_FIT_STEP) without a GPU: the header and the ctypes mirror of nfb_fit_rows_grad, every
argument check of the entry and of nerf.FusedFitter before any CUDA call, and the host restatement of the pose-row order
(pose_rows_fp32, which test_fit_gpu.py holds the kernel to bit for bit) against the order written out literally and against
float64."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "nfb.h")
API = os.path.join(ROOT, "4d-facial-avatars_b200", "csrc", "nfb_api.cu")
F32 = np.float32


def camera_dirs(pixel_rc, fx, fy, wcx, hcy):
    """cx = (col - wcx) / fx, cy = -((row - hcy) / fy), every operation one FP32 rounding (the sampler's helper)."""
    rc = np.asarray(pixel_rc).reshape(-1, 2)
    cx = (rc[:, 1].astype(F32) - F32(wcx)) / F32(fx)
    cy = -((rc[:, 0].astype(F32) - F32(hcy)) / F32(fy))
    return cx.astype(F32), cy.astype(F32)


def slot_terms(cx, cy, go, gd):
    """[rays, 12] FP32 terms of the 3x4 pose row per ray: (dd * cx, dd * cy, -dd, do) per row q (None: zero columns)."""
    t = np.zeros((cx.shape[0], 12), dtype=F32)
    for q in range(3):
        if gd is not None:
            t[:, 4 * q] = gd[:, q] * cx
            t[:, 4 * q + 1] = gd[:, q] * cy
            t[:, 4 * q + 2] = -gd[:, q]
        if go is not None:
            t[:, 4 * q + 3] = go[:, q]
    return t


def pose_rows_fp32(img, n, n_rows, pixel_rc, go, gd, intr, H, W, pose0=None, gexpr=None, expr0=None):
    """The documented order of nfb_fit_rows_grad (include/nfb.h) in FP32 with numpy: per slot, 256 thread-strided sequential
    sums, a halving tree, then the rows in ascending k.  intr = (fx, fy, cx0, cy0) as float64.  Returns (pose rows, expression
    rows, per-slot sums)."""
    fx, fy = F32(intr[0]), F32(intr[1])
    wcx, hcy = F32(float(W) * intr[2]), F32(float(H) * intr[3])
    K = len(img)
    go = None if go is None else np.asarray(go, dtype=F32).reshape(K * n, 3)
    gd = None if gd is None else np.asarray(gd, dtype=F32).reshape(K * n, 3)
    cx, cy = camera_dirs(pixel_rc, fx, fy, wcx, hcy)
    slots = np.zeros((K, 12), dtype=F32)
    with np.errstate(invalid="ignore", over="ignore"):
        for k in range(K):
            s = slice(k * n, (k + 1) * n)
            terms = slot_terms(cx[s], cy[s], None if go is None else go[s], None if gd is None else gd[s])
            part = np.zeros((256, 12), dtype=F32)
            for j in range(0, n, 256):  # thread t adds ray j + t: one vector add per stride, in ascending j
                blk = terms[j:j + 256]
                part[:blk.shape[0]] = part[:blk.shape[0]] + blk
            s_ = 128
            while s_ >= 1:
                part[:s_] = part[:s_] + part[s_:2 * s_]
                s_ //= 2
            slots[k] = part[0]
        G = np.zeros((n_rows, 12), dtype=F32) if pose0 is None else np.array(pose0, dtype=F32)
        E = None if expr0 is None else np.array(expr0, dtype=F32)
        for k, r in enumerate(img):
            if 0 <= r < n_rows:
                G[r] = G[r] + slots[k]
                if E is not None:
                    E[r] = E[r] + np.asarray(gexpr, dtype=F32)[k]
    return G, E, slots


def pose_rows_literal(img, n, n_rows, pixel_rc, go, gd, intr, H, W):
    """The same order as the header words it, one scalar FP32 operation at a time (small n only)."""
    fx, fy = F32(intr[0]), F32(intr[1])
    wcx, hcy = F32(float(W) * intr[2]), F32(float(H) * intr[3])
    G = np.zeros((n_rows, 12), dtype=F32)
    for k, r in enumerate(img):
        partial = [[F32(0.0)] * 12 for _ in range(256)]
        for t in range(256):
            for j in range(t, n, 256):
                i = k * n + j
                row, col = int(pixel_rc[i][0]), int(pixel_rc[i][1])
                cx = F32(F32(F32(col) - wcx) / fx)
                cy = -F32(F32(F32(row) - hcy) / fy)
                for q in range(3):
                    dd, do = F32(gd[i][q]), F32(go[i][q])
                    partial[t][4 * q] = F32(partial[t][4 * q] + F32(dd * cx))
                    partial[t][4 * q + 1] = F32(partial[t][4 * q + 1] + F32(dd * cy))
                    partial[t][4 * q + 2] = F32(partial[t][4 * q + 2] + (-dd))
                    partial[t][4 * q + 3] = F32(partial[t][4 * q + 3] + do)
        s = 128
        while s >= 1:
            for t in range(s):
                partial[t] = [F32(a + b) for a, b in zip(partial[t], partial[t + s])]
            s //= 2
        if 0 <= r < n_rows:
            G[r] = [F32(a + b) for a, b in zip(G[r], partial[0])]
    return G


def gamma(m):
    u = 2.0 ** -24
    return m * u / (1 - m * u)


def test_header_declares_the_entry_and_keeps_the_version():
    text = open(HEADER).read()
    assert re.search(r"#define NFB_FIT_STEP 1\b", text)
    assert re.search(r"#define NFB_VERSION 131\b", text)
    decl = re.search(r"int nfb_fit_rows_grad\((.*?)\);", text, re.S).group(1)
    params = [p.strip() for p in re.sub(r"/\*.*?\*/", "", decl, flags=re.S).split(",")]
    assert [p.split()[-1].lstrip("*") for p in params] == [
        "h", "data", "image_index", "K", "n", "pixel_rc", "grad_ray_origins", "grad_ray_directions", "pose_grads",
        "grad_expressions", "expression_grads", "stream"]
    for word in ("ascending k", "s = 128, 64, 32, 16, 8, 4, 2, 1", "NFB_ERR_UNSUPPORTED for K > NFB_MAX_STEP_IMAGES", "Launches: 2"):
        assert word in text, word


def test_ctypes_mirror(built_lib):
    import nerf
    capi = nerf._capi
    assert "nfb_fit_rows_grad" in capi.EXPORTS
    fn = capi.lib.nfb_fit_rows_grad
    assert fn.restype == C.c_int and len(fn.argtypes) == 12
    assert fn.argtypes[1]._type_ is capi.NfbTrainImages
    assert capi.lib.nfb_version() == 131


def test_entry_checks_fire_before_any_cuda_call(built_lib):
    """Every refusal returns before the handle is touched: a fake handle never dereferenced shows it (a dereference of address 8
    would crash the process)."""
    import nerf
    capi = nerf._capi
    lib = capi.lib
    h = C.c_void_p(8)
    p = C.c_void_p(16)
    good = capi.NfbTrainImages(n_images=2, height=4, width=4)
    no_images = capi.NfbTrainImages(n_images=0, height=4, width=4)
    call = lambda *a: lib.nfb_fit_rows_grad(*a, None)  # noqa: E731
    INV, UNS = 1, 2
    assert call(None, C.byref(good), p, 1, 1, p, p, p, p, p, p) == INV
    assert call(h, None, p, 1, 1, p, p, p, p, p, p) == INV
    assert call(h, C.byref(good), None, 1, 1, p, p, p, p, p, p) == INV
    assert call(h, C.byref(good), p, 0, 1, p, p, p, p, p, p) == INV
    assert call(h, C.byref(good), p, 1, 0, p, p, p, p, p, p) == INV
    assert call(h, C.byref(good), p, 1, 2049, p, p, p, p, p, p) == INV
    assert call(h, C.byref(good), p, 65, 1, p, p, p, p, p, p) == UNS
    assert call(h, C.byref(no_images), p, 1, 1, p, p, p, p, p, p) == INV
    assert call(h, C.byref(good), p, 1, 1, None, p, p, p, p, p) == INV      # pose rows without pixel_rc
    assert call(h, C.byref(good), p, 1, 1, p, None, None, p, p, p) == INV   # pose rows without ray gradients
    assert call(h, C.byref(good), p, 1, 1, p, p, p, p, None, p) == INV      # expression rows without their source
    assert call(h, C.byref(good), p, 1, 1, p, p, p, p, p, None) == INV      # an expression source without rows
    assert call(h, C.byref(good), p, 1, 1, None, None, None, None, None, None) == 0  # nothing asked: no call at all
    body = open(API).read()
    body = body[body.index("int nfb_fit_rows_grad("):]
    body = body[:body.index("\n}\n")]
    first_cuda = body.index("NFB_CUDA(")
    assert all(body.index(ret) < first_cuda for ret in re.findall(r"return NFB_(?:ERR_\w+|OK);", body)[:6])


class _NoLaunch:
    def __getattr__(self, name):
        raise AssertionError(f"renderer used ({name}) before the argument checks")


def _bare_fitter():
    from nerf.fused_fit import FusedFitter
    f = FusedFitter.__new__(FusedFitter)
    f.eng = _NoLaunch()
    f.n_images = 3
    f.data = type("D", (), dict(H=8, W=8, background=None))()
    f._graph = None
    return f


def test_fitter_checks_fire_before_any_launch(built_lib):
    import nerf
    mk = lambda: nerf.models.ConditionalBlendshapePaperNeRFModel(  # noqa: E731
        num_encoding_fn_xyz=10, num_encoding_fn_dir=4, include_input_xyz=True, include_input_dir=False)
    mc, mf = mk(), mk()  # CPU models: a check that came after the renderer would fail with another error
    imgs, boxes, intr = torch.zeros(3, 8, 8, 3), [(0, 8, 0, 8)] * 3, [10.0, 10.0, 0.5, 0.5]
    poses, ex, lat = torch.zeros(3, 12), torch.zeros(3, 76), torch.zeros(3, 32)
    F = nerf.FusedFitter
    with pytest.raises(ValueError, match="nothing to fit"):
        F(mc, mf, imgs, boxes, intr, poses, ex, lat, fit=())
    with pytest.raises(ValueError, match="fit takes"):
        F(mc, mf, imgs, boxes, intr, poses, ex, lat, fit=("pose", "weights"))
    with pytest.raises(ValueError, match="precision"):
        F(mc, mf, imgs, boxes, intr, poses, ex, lat, precision="fastest")
    with pytest.raises(ValueError, match="poses"):
        F(mc, mf, imgs, boxes, intr, torch.zeros(3, 9), ex, lat)
    with pytest.raises(ValueError, match="poses"):
        F(mc, mf, imgs, boxes, intr, poses, torch.zeros(3, 75), lat)
    with pytest.raises(ValueError, match="poses"):
        F(mc, mf, imgs, boxes, intr, poses, ex, torch.zeros(2, 32))
    f = _bare_fitter()
    for args, kw, msg in (
            (([], 4), {}, "K"), ((list(range(65)), 4), {}, "K"), (([0], 0), {}, "n_per_image"), (([0], 2049), {}, "n_per_image"),
            (([0], 65), {}, "n_per_image"), (([0, 3], 4), {}, "out of range"), (([-1], 4), {}, "out of range"),
            (([0], 4), dict(max_rounds=0), "max_rounds"), (([0, 1], 4), dict(draws=torch.zeros(2 * 32 * 4 - 1, dtype=torch.float64)), "draws")):
        for method in (f.step, f.gradients):
            with pytest.raises(ValueError, match=msg):
                method(*args, **kw)
    for k, n, kw in ((0, 4, {}), (65, 4, {}), (1, 0, {}), (1, 65, {}), (1, 4, dict(has_background=True))):
        with pytest.raises(ValueError):
            f.capture(k, n, **kw)
    with pytest.raises(RuntimeError, match="capture"):
        f.step_graph([0])


@pytest.mark.parametrize("K,n,seed", [(1, 1, 0), (2, 300, 1), (3, 257, 2)])
def test_pose_row_restatement_is_the_documented_order(K, n, seed):
    """pose_rows_fp32 (vectorised, what the GPU test holds the kernel to) equals the header's order written out one scalar
    operation at a time, bit for bit, and lies within gamma(n + 2) * sum|term| of the float64 sum; repeats accumulate, an index
    out of range adds nothing."""
    rng = np.random.default_rng(seed)
    H, W, n_rows = 64, 48, 4
    intr = (57.3, 61.9, 0.47, 0.52)
    img = [int(v) for v in rng.integers(-1, n_rows + 1, K)]
    rc = np.stack([rng.integers(0, H, K * n), rng.integers(0, W, K * n)], axis=1).astype(np.int32)
    scale = (10.0 ** rng.integers(-6, 1, (K * n, 1))).astype(F32)
    go = (rng.standard_normal((K * n, 3)).astype(F32) * scale).astype(F32)
    gd = (rng.standard_normal((K * n, 3)).astype(F32) * scale).astype(F32)
    got, _, slots = pose_rows_fp32(img, n, n_rows, rc, go, gd, intr, H, W)
    assert np.array_equal(got, pose_rows_literal(img, n, n_rows, rc, go, gd, intr, H, W))
    cx, cy = camera_dirs(rc, intr[0], intr[1], F32(W * intr[2]), F32(H * intr[3]))
    terms = slot_terms(cx, cy, go, gd).astype(np.float64)
    for k in range(K):
        t = terms[k * n:(k + 1) * n]
        assert (np.abs(slots[k] - t.sum(0)) <= gamma(n + 2) * np.abs(t).sum(0)).all()
    for r in range(n_rows):
        ks = [k for k in range(K) if img[k] == r]
        want = sum((slots[k].astype(np.float64) for k in ks), np.zeros(12))
        assert (np.abs(got[r] - want) <= gamma(len(ks) + 1) * sum((np.abs(slots[k]).astype(np.float64) for k in ks), np.zeros(12))).all()
        if not ks:
            assert not got[r].any()
