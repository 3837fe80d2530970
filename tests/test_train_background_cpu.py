"""A learned background (NFB_TRAIN_BACKGROUND) without a GPU: the header and the ctypes mirror of nfb_background_rows_grad and
nfb_loss_background_grad, every argument check of the entries and of FusedTrainer before any CUDA call, and the host
restatements of both documented orders (background_rows_fp32, loss_background_fp32: what test_train_background_gpu.py holds the
kernels to bit for bit) against the orders written out one scalar at a time and against float64."""
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


def gamma(m):
    u = 2.0 ** -24
    return m * u / (1 - m * u)


def pixel_keys(pixel_rc, H, W):
    """Table row of every ray, row * W + col (the sampler's gather index), -1 outside the table."""
    rc = np.asarray(pixel_rc, dtype=np.int64).reshape(-1, 2)
    ok = (rc[:, 0] >= 0) & (rc[:, 0] < H) & (rc[:, 1] >= 0) & (rc[:, 1] < W)
    return np.where(ok, rc[:, 0] * W + rc[:, 1], -1)


def background_rows_fp32(pixel_rc, H, W, g_render, g_loss=None, table0=None):
    """The documented order of nfb_background_rows_grad in FP32 with numpy: g_r = g_render[r] (+ g_loss[r], one rounding) added
    onto row(r) in ascending r.  Vectorised by occurrence: the j-th ray of every pixel is added in pass j, and the rays of one
    pass name distinct pixels, so each pass is one vector add.  Returns [H*W, 3]."""
    key = pixel_keys(pixel_rc, H, W)
    g = np.asarray(g_render, dtype=F32).reshape(-1, 3)
    with np.errstate(invalid="ignore", over="ignore"):
        if g_loss is not None:
            g = (g + np.asarray(g_loss, dtype=F32).reshape(-1, 3)).astype(F32)
        T = np.zeros((H * W, 3), dtype=F32) if table0 is None else np.array(table0, dtype=F32).reshape(H * W, 3)
        occ = np.zeros(key.shape[0], dtype=np.int64)  # how many earlier rays name the same pixel
        seen = {}
        for r, kk in enumerate(key.tolist()):
            if kk >= 0:
                occ[r] = seen.get(kk, 0)
                seen[kk] = occ[r] + 1
        for j in range(int(occ.max()) + 1 if key.size else 0):
            sel = (occ == j) & (key >= 0)
            T[key[sel]] = T[key[sel]] + g[sel]
    return T


def background_rows_literal(pixel_rc, H, W, g_render, g_loss=None):
    """The same order as the header words it, one scalar FP32 operation at a time (small n only)."""
    T = [[F32(0.0)] * 3 for _ in range(H * W)]
    for r, (row, col) in enumerate(np.asarray(pixel_rc).reshape(-1, 2).tolist()):
        if not (0 <= row < H and 0 <= col < W):
            continue
        for c in range(3):
            g = F32(g_render[r][c]) if g_loss is None else F32(F32(g_render[r][c]) + F32(g_loss[r][c]))
            T[row * W + col][c] = F32(T[row * W + col][c] + g)
    return np.array(T, dtype=F32)


def loss_background_fp32(bg, target, w_last, n_total, weight, loss0=0.0):
    """The documented order of nfb_loss_background_grad in FP32: s = weight * (1 / n_total); per ray d, e = (d0 d0 + d1 d1) +
    d2 d2, grad_bg = (2 d) (s w), grad_w = s e; the terms w e summed by 1024 thread-strided sums, the xor butterfly per warp and
    the 32 warp sums in order; loss0 + S * s.  Returns (grad_bg, grad_w, loss)."""
    bg, t = np.asarray(bg, dtype=F32).reshape(-1, 3), np.asarray(target, dtype=F32).reshape(-1, 3)
    w = np.asarray(w_last, dtype=F32).reshape(-1)
    n = w.shape[0]
    s = F32(F32(weight) * F32(F32(1.0) / F32(n_total)))
    with np.errstate(invalid="ignore", over="ignore"):
        d = (bg - t).astype(F32)
        e = ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]).astype(F32) + (d[:, 2] * d[:, 2]).astype(F32)).astype(F32)
        g_bg = ((F32(2.0) * d) * (s * w)[:, None]).astype(F32)
        g_w = (s * e).astype(F32)
        term = (w * e).astype(F32)
        acc = np.zeros(1024, dtype=F32)
        for j in range(0, n, 1024):
            blk = term[j:j + 1024]
            acc[:blk.shape[0]] = acc[:blk.shape[0]] + blk
        lanes = acc.reshape(32, 32)
        lane = np.arange(32)
        for o in (16, 8, 4, 2, 1):
            lanes = (lanes + lanes[:, lane ^ o]).astype(F32)
        tot = F32(0.0)
        for k in range(32):
            tot = F32(tot + lanes[k, 0])
        loss = F32(F32(loss0) + F32(tot * s))
    return g_bg, g_w, loss


def loss_background_literal(bg, target, w_last, n_total, weight):
    """nfb_loss_background_grad's loss as the header words it, scalar by scalar."""
    s = F32(F32(weight) * F32(F32(1.0) / F32(n_total)))
    n = len(w_last)
    part = [F32(0.0)] * 1024
    for t in range(1024):
        for r in range(t, n, 1024):
            d = [F32(F32(bg[r][c]) - F32(target[r][c])) for c in range(3)]
            e = F32(F32(F32(d[0] * d[0]) + F32(d[1] * d[1])) + F32(d[2] * d[2]))
            part[t] = F32(part[t] + F32(F32(w_last[r]) * e))
    warps = []
    for wp in range(32):
        v = part[32 * wp:32 * wp + 32]
        for o in (16, 8, 4, 2, 1):
            v = [F32(v[l] + v[l ^ o]) for l in range(32)]
        warps.append(v[0])
    tot = F32(0.0)
    for x in warps:
        tot = F32(tot + x)
    return F32(tot * s)


def test_header_declares_the_entries_and_keeps_the_version():
    text = open(HEADER).read()
    assert re.search(r"#define NFB_TRAIN_BACKGROUND 1\b", text)
    assert re.search(r"#define NFB_VERSION 131\b", text)
    for name, want in (("nfb_background_rows_grad", ["h", "pixel_rc", "n_rays", "height", "width", "grad_bg_render", "grad_bg_loss",
                                                    "table_grads", "stream"]),
                       ("nfb_loss_background_grad", ["h", "bg_rays", "target", "w_last", "n_rays", "n_total", "weight", "grad_bg_rays",
                                                    "grad_w_last", "loss", "stream"])):
        decl = re.search(rf"int {name}\((.*?)\);", text, re.S).group(1)
        params = [p.strip() for p in re.sub(r"/\*.*?\*/", "", decl, flags=re.S).split(",")]
        assert [p.split()[-1].lstrip("*") for p in params] == want, name
    for word in ("in ascending r", "no atomics", "(2 * d[c]) * (s * w_last[r])", "offsets 16, 8, 4, 2, 1", "Launches: 1."):
        assert word in text, word


def test_ctypes_mirror(built_lib):
    import nerf
    capi = nerf._capi
    for name, nargs in (("nfb_background_rows_grad", 9), ("nfb_loss_background_grad", 11)):
        assert name in capi.EXPORTS
        fn = getattr(capi.lib, name)
        assert fn.restype == C.c_int and len(fn.argtypes) == nargs, name
    assert capi.lib.nfb_loss_background_grad.argtypes[6] is C.c_float
    assert capi.lib.nfb_version() == 131


def _refusals_precede_cuda(name, count):
    body = open(API).read()
    body = body[body.index(f"int {name}("):]
    body = body[:body.index("\n}\n")]
    first_cuda = body.index("NFB_CUDA(")
    rets = re.findall(r"return NFB_(?:ERR_\w+|OK);", body)
    assert len(rets) >= count
    assert all(body.index(ret) < first_cuda for ret in rets[:count])


def test_entry_checks_fire_before_any_cuda_call(built_lib):
    """Every refusal returns before the handle is touched: a fake handle never dereferenced shows it."""
    import nerf
    lib = nerf._capi.lib
    h, p = C.c_void_p(8), C.c_void_p(16)
    INV = 1
    rows = lambda *a: lib.nfb_background_rows_grad(*a, None)  # noqa: E731
    assert rows(None, p, 4, 8, 8, p, p, p) == INV
    assert rows(h, None, 4, 8, 8, p, p, p) == INV
    assert rows(h, p, -1, 8, 8, p, p, p) == INV
    assert rows(h, p, 4, 0, 8, p, p, p) == INV
    assert rows(h, p, 4, 8, 0, p, p, p) == INV
    assert rows(h, p, 4, 65536, 65536, p, p, p) == INV     # more pixels than an int index holds
    assert rows(h, p, 4, 8, 8, None, p, p) == INV
    assert rows(h, p, 4, 8, 8, p, p, None) == INV
    assert rows(h, p, 0, 8, 8, p, None, p) == 0            # no rays: nothing added, no call at all
    loss = lambda *a: lib.nfb_loss_background_grad(*a, None)  # noqa: E731
    for i in range(11):
        if i in (4, 5, 6):
            continue
        args = [h, p, p, p, 4, 8, 0.001, p, p, p]
        if i < 10:
            args[i] = None
            assert loss(*args) == INV, i
    assert loss(h, p, p, p, -1, 8, 0.001, p, p, p) == INV
    assert loss(h, p, p, p, 4, 3, 0.001, p, p, p) == INV      # n_total < n_rays
    assert loss(h, p, p, p, 0, 0, 0.001, p, p, p) == INV      # n_total <= 0
    assert loss(h, p, p, p, 0, 8, 0.001, p, p, p) == 0        # an empty shard: no call
    _refusals_precede_cuda("nfb_background_rows_grad", 3)
    _refusals_precede_cuda("nfb_loss_background_grad", 2)


class _NoLaunch:
    def __getattr__(self, name):
        raise AssertionError(f"renderer used ({name}) before the argument checks")


def test_trainer_checks_fire_before_any_launch(built_lib):
    import nerf
    from nerf.fused_train import FusedTrainer
    mk = lambda: nerf.models.ConditionalBlendshapePaperNeRFModel(  # noqa: E731
        num_encoding_fn_xyz=10, num_encoding_fn_dir=4, include_input_xyz=True, include_input_dir=False)
    mc, mf = mk(), mk()  # CPU models: a check after the renderer would fail with another error
    with pytest.raises(ValueError, match=r"\[H,W,3\]"):
        FusedTrainer(mc, mf, 2, background=torch.zeros(8, 8))
    with pytest.raises(ValueError, match=r"\[H,W,3\]"):
        FusedTrainer(mc, mf, 2, background=torch.zeros(8, 8, 4))
    with pytest.raises(ValueError, match="background="):
        FusedTrainer(mc, mf, 2, background_loss=0.001)
    with pytest.raises(ValueError, match=">= 0"):
        FusedTrainer(mc, mf, 2, background=torch.zeros(8, 8, 3), background_loss=-1.0)
    t = FusedTrainer.__new__(FusedTrainer)
    t.eng = _NoLaunch()
    t.background = torch.zeros(8, 6, 3)
    t.latent_codes = torch.zeros(4, 32)
    for call in (lambda: t.step(None, None, None, None, 0), lambda: t.gradients(None, None, None, None, 0), lambda: t.capture(64),
                 lambda: t.step_graph(None, None, None, None, 0)):
        with pytest.raises(ValueError, match="step_images"):
            call()
    D = lambda bg, H=8, W=6: type("D", (), dict(H=H, W=W, n_images=3, background=bg))()  # noqa: E731
    with pytest.raises(ValueError, match="carry"):
        t._check_images(D(torch.zeros(8, 6, 3)), 2, 16, 1)
    with pytest.raises(ValueError, match="frames"):
        t._check_images(D(None, 6, 8), 2, 16, 1)
    assert t._check_images(D(None), 2, 16, 1) == 0
    for method in (t.step_images, t.capture_images):
        with pytest.raises(ValueError, match="carry"):
            method(D(torch.zeros(8, 6, 3)), [0, 1] if method == t.step_images else 2, 16)


@pytest.mark.parametrize("n,H,W,seed", [(1, 4, 4, 0), (7, 3, 5, 1), (300, 6, 7, 2), (2500, 16, 16, 3)])
def test_row_restatement_is_the_documented_order(n, H, W, seed):
    """background_rows_fp32 equals the header's order written out scalar by scalar, bit for bit, with and without the loss term,
    with repeated pixels, out-of-range entries and a NaN; each row lies within gamma(m) * sum|g| of float64 (m: its hits)."""
    rng = np.random.default_rng(seed)
    rc = np.stack([rng.integers(-1, H + 1, n), rng.integers(-1, W + 1, n)], axis=1).astype(np.int32)
    rc[::5] = rc[0]  # a pixel hit many times
    scale = (10.0 ** rng.integers(-6, 1, (n, 1))).astype(F32)
    gr = (rng.standard_normal((n, 3)) * scale).astype(F32)
    gl = (rng.standard_normal((n, 3)) * scale * 0.1).astype(F32)
    if n > 3:
        gr[3, 1] = np.nan
    for g_loss in (None, gl):
        got = background_rows_fp32(rc, H, W, gr, g_loss)
        lit = background_rows_literal(rc, H, W, gr, g_loss)
        assert np.array_equal(got, lit, equal_nan=True)
        key = pixel_keys(rc, H, W)
        g64 = gr.astype(np.float64) + (0.0 if g_loss is None else g_loss.astype(np.float64))
        for px in range(H * W):
            hits = np.nonzero(key == px)[0]
            if hits.size == 0:
                assert not got[px].any()
                continue
            if np.isnan(g64[hits]).any():
                assert np.isnan(got[px]).any()
                continue
            want = g64[hits].sum(0)
            assert (np.abs(got[px] - want) <= gamma(2 * hits.size) * np.abs(g64[hits]).sum(0) + 1e-45).all(), px
        if n > 3 and 0 <= rc[3, 0] < H and 0 <= rc[3, 1] < W:  # the NaN stays on its own pixel
            assert np.isnan(got[key[3], 1]) and np.isfinite(np.delete(got, key[3], axis=0)).all()


@pytest.mark.parametrize("n,seed", [(1, 0), (37, 1), (1500, 2)])
def test_loss_restatement_is_the_documented_order(n, seed):
    """loss_background_fp32's loss equals the header's order written out scalar by scalar, and lies within the gamma bound of
    float64; its gradients are the autograd formula in float64 to one rounding each."""
    rng = np.random.default_rng(seed)
    bg, t = rng.random((n, 3)).astype(F32), rng.random((n, 3)).astype(F32)
    w = rng.random(n).astype(F32)
    n_total, weight = 4 * n, 0.001
    g_bg, g_w, loss = loss_background_fp32(bg, t, w, n_total, weight)
    assert loss == loss_background_literal(bg, t, w, n_total, weight)
    d = bg.astype(np.float64) - t.astype(np.float64)
    e = (d * d).sum(1)
    want = weight / n_total * float((w * e).sum())
    assert abs(float(loss) - want) <= gamma(n + 40) * want
    assert np.allclose(g_bg, weight / n_total * 2 * d * w[:, None], rtol=1e-6, atol=0)
    assert np.allclose(g_w, weight / n_total * e, rtol=1e-6, atol=0)
